"""The slicing step of dataset preparation: recordings cut at their pauses into loudness-normalised int16 chunks.

Mirror of `AudioService.slicer` (reference src/service/audio.py:142-183) and of the `Slicer` it drives
(src/audiokit/slicer/slicer.py).  For every file the reference
  1. decodes it to mono float32 at 32 kHz (`load_audio`) and skips it when it is empty,
  2. takes the RMS of 1280-sample frames every 320 samples (`Slicer.get_rms`),
  3. walks the frames for pauses (`rms < threshold`) and turns them into silence tags (slicer.py:53-131),
  4. cuts the samples between the tags into chunks (slicer.py:133-147), and for every chunk
  5. m = max |chunk|;  m > 1: chunk /= m;  chunk = (chunk / m * (normalize_max * alpha_mix)) + (1 - alpha_mix) * chunk
     (m is still the old max: a chunk with m > 1 is divided twice), written as int16(chunk * 32767) to
     `<name>_<start:010d>_<end:010d>.wav`.

Same files in, same files out.  Here rows are grouped longest-first into zero-padded batches that cross to the device once;
`evk_frame_rms` does step 2 for the batch and only the RMS comes back (one float per 320 samples); step 3 runs on the host
over the silent runs instead of over every frame; `evk_slice_normalize` does step 5 for every chunk of the batch in one call on
the samples that are still on the device, and the int16 buffer comes back once.  Decoding and the wav writes stay with the
caller's `load_audio` and scipy.

The device RMS is the float64 value rounded once, which numpy's float32 mean only approximates (to about 1e-7), so a frame
whose RMS is within that of the threshold, or two candidate cut frames that close to each other, can be decided differently.
tests/golden/slicer.pt records the margins of the pinned recordings.

Reference behaviour that is kept:
  * `samples.shape[0] <= self.min_length` compares samples with frames (400 at the defaults).  `Slicer.slice` then returns
    `[waveform]`, which the service's `for chunk, start, end in ...` cannot unpack; its `except` swallows that.  Such a file
    writes nothing and is not in `data`; here its name is also in `failed`.
  * The reported end of a chunk is `end_frame * hop` and goes into the file name; it may exceed the recording's length, while
    the samples stop at the length.
  * A chunk can be empty (it starts at the recording's last sample; only a NaN frame gets a cut there).  `np.abs(chunk).max()`
    then raises after the file's earlier chunks were written: those are written, none after it, and the file is in `failed`
    and not in `data`.
  * No silence tag gives one chunk `[waveform, 0, total_frames * hop]`.
  * A chunk of digital silence (m == 0) is 0 / 0 = NaN throughout, which converts to int16 0: the file is written.
"""
import os

import numpy as np
import torch
from scipy.io import wavfile

from . import lib, ops
from .normalize_ssl import _pack

SR = 32000
SLICE_OK, SLICE_SILENT, SLICE_NONFINITE = 0, 1, 2        # evk_slice_status
MAX_SAMPLES = 1 << 26                                    # padded samples of one batch: 256 MiB of float32 on the device
SUCCESS = "Success"                                      # ResponseStatus.SUCCESS (reference src/utils/response.py)


class Slicer(object):
    def __init__(self, sr, threshold=-34.0, min_length=4000, min_interval=300, hop_size=10, max_sil_kept=500):
        """slicer.py:8-31: times in ms, threshold in dB; the derived fields are in frames except hop_size and win_size (samples)"""
        if not min_length >= min_interval >= hop_size:
            raise ValueError("The following condition must be satisfied: min_length >= min_interval >= hop_size")
        if not max_sil_kept >= hop_size:
            raise ValueError("The following condition must be satisfied: max_sil_kept >= hop_size")
        min_interval = sr * min_interval / 1000
        self.threshold = 10 ** (threshold / 20.0)
        self.hop_size = round(sr * hop_size / 1000)
        self.win_size = min(round(min_interval), 4 * self.hop_size)
        self.min_length = round(sr * min_length / 1000 / self.hop_size)
        self.min_interval = round(min_interval / self.hop_size)
        self.max_sil_kept = round(sr * max_sil_kept / 1000 / self.hop_size)

    def num_frames(self, n):
        """frames `get_rms` makes of n samples"""
        return 1 + (n + 2 * (self.win_size // 2) - self.win_size) // self.hop_size

    def scan(self, rms):
        """slicer.py:53-131 on the RMS of one recording -> sil_tags, the list of (first, last) removed frames.  The reference
        visits every frame; its state only changes where a silent run ends, and a run can only produce a tag when it starts
        at frame 0 or is at least min_interval long, so only those runs are visited."""
        n, msk = int(rms.shape[0]), self.max_sil_kept
        edge = np.zeros(n + 2, dtype=np.int8)
        edge[1:-1] = rms < self.threshold
        d = np.diff(edge)
        starts, ends = np.flatnonzero(d == 1), np.flatnonzero(d == -1)       # silent runs [s, e); e is the next loud frame
        keep = (starts == 0) | (ends - starts >= self.min_interval)
        tags, clip_start = [], 0

        def argmin(lo, hi):                                                  # rms_list[lo:hi + 1].argmin() + lo
            return int(rms[lo:hi + 1].argmin()) + lo

        for s, i in zip(starts[keep].tolist(), ends[keep].tolist()):
            if i == n:                                                       # trailing silence
                if n - s >= self.min_interval:
                    tags.append((argmin(s, min(n, s + msk)), n + 1))
                break
            leading = s == 0 and i > msk
            middle = i - s >= self.min_interval and i - clip_start >= self.min_length
            if not leading and not middle:
                continue
            if i - s <= msk:
                pos = argmin(s, i)
                tags.append((0, pos) if s == 0 else (pos, pos))
                clip_start = pos
            else:
                pos_l, pos_r = argmin(s, s + msk), argmin(i - msk, i)
                if i - s <= msk * 2 and s != 0:
                    pos = argmin(i - msk, s + msk)
                    pos_l, pos_r = min(pos_l, pos), max(pos_r, pos)
                tags.append((0, pos_r) if s == 0 else (pos_l, pos_r))
                clip_start = pos_r
        return tags

    def ranges(self, tags, total_frames):
        """slicer.py:133-147: (start, end) in samples of every chunk, as reported: end may exceed the length"""
        hop = self.hop_size
        if not tags:
            return [(0, int(total_frames * hop))]
        out = []
        if tags[0][0] > 0:
            out.append((0, int(tags[0][0] * hop)))
        for a, b in zip(tags[:-1], tags[1:]):
            out.append((int(a[1] * hop), int(b[0] * hop)))
        if tags[-1][1] < total_frames:
            out.append((int(tags[-1][1] * hop), int(total_frames * hop)))
        return out

    def _batches(self, clips, max_samples):
        """clips: checked float32 rows.  Yields (rows of the batch, device samples [nb, Lm], [(ranges, tags)] per row); rows
        of at most min_length samples are in no batch."""
        order = sorted((i for i in range(len(clips)) if len(clips[i]) > self.min_length), key=lambda i: -len(clips[i]))
        if not order:
            return
        lib.init()
        dev = torch.device("cuda", torch.cuda.current_device())
        i = 0
        while i < len(order):
            Lm = len(clips[order[i]])
            nb = max(1, min(65535, max_samples // Lm))
            grp = order[i:i + nb]
            i += nb
            x, lens_d, _ = _pack(clips, grp, dev)
            rms = ops.frame_rms(x, lens_d, self.win_size, self.hop_size).cpu().numpy()
            res = []
            for r, j in enumerate(grp):
                frames = self.num_frames(len(clips[j]))
                tags = self.scan(rms[r, :frames])
                res.append((self.ranges(tags, frames), tags))
            yield grp, x, res

    def slice_batch(self, clips, max_samples=MAX_SAMPLES):
        """clips: list of 1-D float32-convertible arrays -> per clip (ranges, sil_tags), ranges the reported (start_sample,
        end_sample) of every chunk (the samples are clip[start:min(len, end)]); None for a clip of at most min_length samples,
        where `slice` returns `[waveform]`."""
        clips = [check_clip(a, f"clip {i}", max_samples) for i, a in enumerate(clips)]
        out = [None] * len(clips)
        for grp, _, res in self._batches(clips, max_samples):
            for j, r in zip(grp, res):
                out[j] = r
        return out

    def slice(self, waveform):
        """slicer.py:43-147 for one mono recording -> [[chunk, start, end], ...] with chunk a view of waveform, or [waveform]
        when it has at most min_length samples"""
        if len(waveform.shape) > 1:
            raise ValueError(f"Slicer.slice takes mono samples, got shape {waveform.shape}")
        res = self.slice_batch([waveform])[0]
        if res is None:
            return [waveform]
        return [[waveform[s:min(waveform.shape[0], e)], s, e] for s, e in res[0]]


def check_clip(a, name, max_samples=MAX_SAMPLES):
    """-> a as contiguous float32, or ValueError for what the device cannot take"""
    a = np.asarray(a)
    if a.ndim != 1:
        raise ValueError(f"{name}: expected mono samples, got shape {a.shape}")
    if a.dtype.kind not in "fiu":
        raise ValueError(f"{name}: samples of dtype {a.dtype} do not convert to float32")
    if a.size > max_samples:
        raise ValueError(f"{name}: {a.size} samples are more than one batch holds ({max_samples})")
    return np.ascontiguousarray(a, dtype=np.float32)


def slice_and_normalize(slicer, clips, normalize_max=0.9, alpha_mix=0.25, max_samples=MAX_SAMPLES):
    """Steps 2-5 of the module docstring for a list of recordings -> per clip None (at most min_length samples) or
    dict(ranges, tags, chunks, status, empty): chunks the int16 arrays of ranges[:len(chunks)], status their evk_slice_status,
    empty True when chunk len(chunks) has no samples (the reference fails there, so no later chunk is made)."""
    clips = [check_clip(a, f"clip {i}", max_samples) for i, a in enumerate(clips)]
    c1, c2 = np.float32(normalize_max * alpha_mix), np.float32(1 - alpha_mix)
    out = [None] * len(clips)
    for grp, x, res in slicer._batches(clips, max_samples):
        Lm = x.shape[1]
        table, owner = [], []
        for r, (j, (ranges, tags)) in enumerate(zip(grp, res)):
            out[j] = dict(ranges=ranges, tags=tags, chunks=[], status=[], empty=False)
            for s, e in ranges:
                e = min(len(clips[j]), e)
                if e <= s:
                    out[j]["empty"] = True
                    break
                table.append((r * Lm + s, e - s))
                owner.append(j)
        if not table:
            continue
        t = np.asarray(table, dtype=np.int64)
        y, _, status = ops.slice_normalize(x.view(-1), torch.from_numpy(t).to(x.device), int(t[:, 1].max()), c1, c2)
        y, status = y.cpu().numpy(), status.cpu().tolist()
        for (off, n), j, st in zip(table, owner, status):
            out[j]["chunks"].append(y[off:off + n].copy())
            out[j]["status"].append(st)
    return out


def write_slices(files, out_dir, load_audio, threshold=-34, min_length=4000, min_interval=300, hop_size=10, max_silent_kept=500,
                 normalize_max=0.9, alpha_mix=0.25, sr=SR, max_samples=MAX_SAMPLES):
    """`AudioService.slicer` body (audio.py:155-183) for `files`, writing `<name>_<start:010d>_<end:010d>.wav` into out_dir.
    load_audio(path, sr) is the caller's decoder (the reference's src.utils.audio.load_audio: ffmpeg, mono float32); what it
    raises is not caught.  Samples that are not 1-D, do not convert to float32 or exceed max_samples raise ValueError naming
    the file before any GPU work.  Files are written in the order of `files`.  Returns (data, failed): data is {name: SUCCESS},
    the dict the service returns; failed lists the names the reference's `except` swallows (see the module docstring), which
    are not in data.  Empty audio is skipped and is in neither."""
    slicer = Slicer(sr=sr, threshold=int(threshold), min_length=int(min_length), min_interval=int(min_interval),
                    hop_size=int(hop_size), max_sil_kept=int(max_silent_kept))
    names, clips = [], []
    for file in files:
        audio = check_clip(load_audio(file, sr), str(file), max_samples)
        if audio.shape[0] == 0:
            continue
        names.append(os.path.basename(file).split(".")[0])
        clips.append(audio)
    data, failed = {}, []
    for name, res in zip(names, slice_and_normalize(slicer, clips, normalize_max, alpha_mix, max_samples)):
        for (start, end), chunk in zip(res["ranges"], res["chunks"]) if res is not None else ():
            wavfile.write(os.path.join(out_dir, "%s_%010d_%010d.wav" % (name, start, end)), sr, chunk)
        if res is None or res["empty"]:
            failed.append(name)
        else:
            data[name] = SUCCESS
    return data, failed
