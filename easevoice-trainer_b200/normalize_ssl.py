"""HuBERT features and 32 kHz int16 waveforms of the dataset preparation step (SURVEY section 8 row f3, ssl half).

Mirror of `Normalize.ssl` (reference src/normalization/normalize.py:131-179): for every line of the refinements list
(`wav_name|language|text`) whose `4-cnhubert/<name>.pt` does not exist yet, `_name2go` takes the decoded 32 kHz samples a and
  1. m = max |a|; m > 2.2: nothing is written (the file still counts as a success)
  2. a32 = (a / m * c1) + c2 * a  and  a32b = (a / m * c1b) + c2b * a  (loudness normalisation, two scales)
  3. a16 = librosa.resample(a32b, orig_sr=32000, target_sr=16000)  (librosa 0.9.2 defaults: resampy's kaiser_best)
  4. ssl = HubertModel(a16[None])["last_hidden_state"].transpose(1, 2)  -> [1, 768, T]
  5. NaN in ssl: nothing is written (the caller still reports success); else 5-wav32k/<name> <- int16(a32) at 32 kHz and
     4-cnhubert/<name>.pt <- ssl.

Same files in, same files out.  Here every utterance takes one device pass: rows are grouped longest-first into zero-padded
batches, the samples cross to the device once, `evk_ssl_normalize` does steps 1-2 for the whole batch, `evk_resample_poly`
step 3, `hubert.HubertModel` (ragged lengths) step 4, and the int16 waveforms and features cross back once.  The reference
runs this on the CPU, rebuilding the model for every file.  Audio decoding stays with the caller (`load_audio`).

Resampling assumption (librosa / resampy are not dependencies): with a ratio of exactly 1/2, resampy's `resample_f` reads its
kaiser_best table (64 zero crossings, 2^16 entries per crossing, rolloff 0.9475937167399596, Kaiser beta 14.769656459379492)
at fractional offset 0 or 1/2 only, at every 32768th entry, so the call is the fixed symmetric FIR of `resample_taps`
  a16[n] = sum_{d=-127..127} h[|d|] a32b[2n + d]   (samples outside the row are 0),
floor(L / 2) outputs, and librosa's fix_length appends one 0 for odd L.
"""
import functools
import os

import numpy as np
import torch
from scipy.io import wavfile

from . import ops
from .normalize_token import format_path

SR = 32000
SSL_OK, SSL_SKIP, SSL_NONFINITE = 0, 1, 2            # evk_ssl_status
_ROLLOFF, _BETA, _HALF = 0.9475937167399596, 14.769656459379492, 128


@functools.lru_cache(maxsize=1)
def resample_taps():
    """-> (h [128] float64: h[j] = 0.5 r sinc(r j / 2) I0(beta sqrt(1 - (j / 128)^2)) / I0(beta), the zero-prefixed fp32 filter
    [256] that evk_resample_poly reads with up = 1, down = 2, n_pre_remove = 64: f[k] = h[|k - 128|] for k >= 1, f[0] = 0)."""
    j = np.arange(_HALF, dtype=np.float64)
    h = 0.5 * _ROLLOFF * np.sinc(_ROLLOFF * j / 2) * np.i0(_BETA * np.sqrt(1.0 - (j / _HALF) ** 2)) / np.i0(_BETA)
    f = np.zeros(2 * _HALF, dtype=np.float64)
    f[1:] = h[np.abs(np.arange(1, 2 * _HALF) - _HALF)]
    return h, f.astype(np.float32)


def _pack(clips, grp, dev):
    """rows of clips[grp] zero-padded to the longest, with their lengths and half lengths appended as int32 bit patterns:
    one host-to-device copy per batch"""
    Lm, nb = len(clips[grp[0]]), len(grp)
    buf = np.zeros(nb * Lm + 2 * nb, dtype=np.float32)
    meta = buf[nb * Lm:].view(np.int32)
    for r, j in enumerate(grp):
        buf[r * Lm:r * Lm + len(clips[j])] = clips[j]
        meta[r], meta[nb + r] = len(clips[j]), len(clips[j]) // 2
    d = torch.from_numpy(buf).to(dev)
    return d[:nb * Lm].view(nb, Lm), d[nb * Lm:nb * Lm + nb].view(torch.int32), d[nb * Lm + nb:].view(torch.int32)


def check_clip(model, a, name="clip"):
    """ValueError for audio `_name2go` cannot take: empty (numpy's max raises) or shorter at 16 kHz than one HuBERT frame."""
    if a.ndim != 1 or a.size == 0:
        raise ValueError(f"{name}: no samples (shape {a.shape})")
    if model.num_frames((a.size + 1) // 2) < 1:
        raise ValueError(f"{name}: {a.size} samples at 32 kHz are shorter than one HuBERT frame (400 samples at 16 kHz)")


@torch.no_grad()
def extract(model, clips, max_batch=32, max_samples=1 << 23):
    """clips: list of 1-D float32 numpy arrays of 32 kHz samples -> one (status, int16 numpy waveform or None, fp32 CPU
    features [1, 768, T] or None) per clip, in order.  status: SSL_OK (both outputs), SSL_SKIP (max |a| > 2.2) or
    SSL_NONFINITE (silent or NaN input, or NaN features).  Batches hold at most max_batch rows and max_samples padded samples."""
    dev = next(iter(model.parameters())).device
    clips = [np.ascontiguousarray(a, dtype=np.float32) for a in clips]
    for i, a in enumerate(clips):
        check_clip(model, a, f"clip {i}")
    taps = torch.from_numpy(resample_taps()[1]).to(dev)
    order = sorted(range(len(clips)), key=lambda i: -len(clips[i]))
    out = [None] * len(clips)
    i = 0
    while i < len(order):
        Lm = len(clips[order[i]])
        nb = max(1, min(max_batch, max_samples // Lm))
        grp = order[i:i + nb]
        i += nb
        x, lens_d, half_d = _pack(clips, grp, dev)
        a32, a32b, status = ops.ssl_normalize(x, lens_d)
        n16 = [(len(clips[j]) + 1) // 2 for j in grp]
        a16 = ops.resample_poly(a32b, taps, 1, 2, 64, (Lm + 1) // 2)
        a16 = ops.rowmask(a16.unsqueeze(-1), half_d).squeeze(-1)      # floor(L / 2) FIR outputs, then fix_length's zero
        st = status.cpu().tolist()
        ok = [r for r in range(len(grp)) if st[r] == SSL_OK]
        feats = None
        if ok:
            sel = torch.tensor(ok, device=dev)
            feats = model(a16.index_select(0, sel), [n16[r] for r in ok])["last_hidden_state"].cpu()
            wav = a32.index_select(0, sel).cpu().numpy()
        for r, j in enumerate(grp):
            out[j] = (st[r], None, None)
        for k, r in enumerate(ok):
            j = grp[r]
            f = feats[k, :model.num_frames(n16[r])].t().unsqueeze(0).contiguous()
            if bool(torch.isnan(f).any()):                                # normalize.py:169-170
                out[j] = (SSL_NONFINITE, None, None)
            else:
                out[j] = (SSL_OK, wav[k, :len(clips[j])].copy(), f)
    return out


def write_hubert_features(refinements_path, wav_dir, hubert_dir, wav32_dir, model, load_audio, max_batch=32, max_samples=1 << 23):
    """`Normalize.ssl` body (normalize.py:131-179) with is_half False, as the reference runs it.  load_audio(path, 32000) is the
    caller's decoder (the reference's src.utils.audio.load_audio: ffmpeg, mono float32).  Lines whose feature file exists
    are skipped; empty or too-short audio raises ValueError naming the file before any GPU work.  Returns the names that
    failed (silent or NaN input, NaN features): nothing was written for them, and the reference still reports success."""
    with open(refinements_path, "r", encoding="utf8") as f:
        lines = f.read().strip("\n").split("\n")
    names, clips, seen = [], [], set()
    for line in lines:
        if not line:
            continue
        wav_name, _language, _text = line.split("|")
        wav_name = os.path.basename(format_path(wav_name))
        if wav_name in seen or os.path.exists(os.path.join(hubert_dir, wav_name + ".pt")):
            continue                                                      # normalize.py:152-153
        seen.add(wav_name)
        path = os.path.join(wav_dir, wav_name)
        a = np.asarray(load_audio(path, SR), dtype=np.float32)
        check_clip(model, a, path)
        names.append(wav_name)
        clips.append(a)
    failed = []
    for name, (st, wav, feat) in zip(names, extract(model, clips, max_batch=max_batch, max_samples=max_samples)):
        if st == SSL_NONFINITE:
            failed.append(name)
        elif st == SSL_OK:
            wavfile.write(os.path.join(wav32_dir, name), SR, wav)
            torch.save(feat, os.path.join(hubert_dir, name + ".pt"))
    return failed
