"""GPU tests of Normalize.ssl on the device (`pytest -m gpu`): the length-aware GroupNorm, evk_attn_pad_fwd past 512 keys, the
loudness-normalisation kernel and the 2:1 resampler against numpy / float64 restatements, ragged HuBERT batches against the
oracle's single-utterance forward, and the `write_hubert_features` drop-in against the files the reference wrote
(tests/golden/normalize_ssl.pt, oracle/pin_normalize_ssl.py)."""
import os

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import hubert_oracle, ssl_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "normalize_ssl.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
TOL_NET = 3e-3


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _net(layers, seed):
    from easevoice_trainer_b200 import hubert
    m = dict(hubert_oracle.HUBERT_BASE, layers=layers)
    P = hubert_oracle.init_params(hubert_oracle.param_spec(m), seed)
    net = hubert.HubertModel({"num_hidden_layers": layers})
    net.load_state_dict(P)
    return net.to(DEV).eval(), P, m


def test_instnorm_lens_against_float64(ops):
    B, T, C = 3, 301, 70
    lens = [301, 120, 1]
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, T, C, generator=g) * 2.0 + 0.5
    gm, bt = 1.0 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    xd, gd, bd = x.to(DEV), gm.to(DEV), bt.to(DEV)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    for gelu in (False, True):
        y = ops.instnorm_cl(xd, gd, bd, gelu_after=gelu, lens=lens_d).cpu()
        for b, n in enumerate(lens):
            if n > 1:                                      # torch's group_norm refuses one value per group
                want = torch.nn.functional.group_norm(x[b:b + 1, :n].transpose(1, 2).double(), C, gm.double(), bt.double(), 1e-5)
                want = want.transpose(1, 2)[0]
                assert rel(y[b, :n], torch.nn.functional.gelu(want) if gelu else want) <= 2e-6, (gelu, b)
            assert bool(torch.isfinite(y[b, :n]).all()) and bool((y[b, n:] == 0).all()), (gelu, b)
        # NULL lens is every frame: the same launch as lens = T for every item
        full = torch.full((B,), T, dtype=torch.int32, device=DEV)
        assert torch.equal(ops.instnorm_cl(xd, gd, bd, gelu_after=gelu), ops.instnorm_cl(xd, gd, bd, gelu_after=gelu, lens=full))
    # statistics of an item do not depend on T or on the padding
    x2 = torch.cat([x, 1e3 * torch.randn(B, 50, C, generator=g)], 1)
    x2[1, 120:] = -7e2
    y2 = ops.instnorm_cl(x2.to(DEV), gd, bd, lens=lens_d).cpu()
    y1 = ops.instnorm_cl(xd, gd, bd, lens=lens_d).cpu()
    for b, n in enumerate(lens):
        assert torch.equal(y2[b, :n], y1[b, :n])


@pytest.mark.parametrize("L", [700, 1500])
def test_attention_pad_past_512_keys(ops, L):
    B, H, D = 3, 12, 768
    lens = [L, L // 3, 513]
    g = torch.Generator().manual_seed(200 + L)
    qkv = torch.randn(B, L, 3 * D, generator=g)
    out = ops.attention_pad(qkv.to(DEV), heads=H, lens=torch.tensor(lens, device=DEV), scale=0.125).cpu()
    assert bool(torch.isfinite(out).all())
    c = qkv.double()
    for b in range(B):
        q, k, v = [c[b, :, i * D:(i + 1) * D].view(L, H, 64).transpose(0, 1) for i in range(3)]
        s = (q @ k[:, :lens[b]].transpose(-1, -2)) * 0.125
        want = (s.softmax(-1) @ v[:, :lens[b]]).transpose(0, 1).reshape(L, D)
        assert rel(out[b, :lens[b]], want[:lens[b]]) <= 1e-3, b


def _ragged_rows(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * 0.3 for n in lengths]


def test_padding_content_does_not_reach_valid_frames(ops):
    net, _, _ = _net(2, 41)
    lengths = [16000, 9001, 4000, 12345]
    rows = _ragged_rows(lengths, 7)
    L = max(lengths)
    zero = torch.zeros(len(rows), L)
    noise = 50.0 * torch.randn(len(rows), L, generator=torch.Generator().manual_seed(8))
    for r, x in enumerate(rows):
        zero[r, :len(x)] = x
        noise[r, :len(x)] = x
    a = net(zero.to(DEV), lengths)["last_hidden_state"].cpu()
    b = net(noise.to(DEV), lengths)["last_hidden_state"].cpu()
    assert bool(torch.isfinite(b).all())
    for r, n in enumerate(lengths):
        T = net.num_frames(n)
        assert torch.equal(a[r, :T], b[r, :T]), r


@pytest.mark.parametrize("layers,seed,lengths", [(2, 41, [16000, 9001, 4000, 12345]), (12, 42, [24000, 8000, 401, 15999])])
def test_ragged_hubert_rows_match_single_utterance_oracle(ops, layers, seed, lengths):
    net, P, m = _net(layers, seed)
    rows = _ragged_rows(lengths, seed + 1)
    x = torch.zeros(len(rows), max(lengths))
    for r, w in enumerate(rows):
        x[r, :len(w)] = w
    out = net(x.to(DEV), lengths)["last_hidden_state"].cpu()
    assert out.shape == (len(rows), net.num_frames(max(lengths)), 768)
    for r, w in enumerate(rows):
        T = net.num_frames(len(w))
        with torch.no_grad():
            want = hubert_oracle.forward(P, w[None], m)[0]
        alone = net(w[None].to(DEV))["last_hidden_state"][0].cpu()
        assert want.shape[0] == T and alone.shape[0] == T
        e_oracle, e_alone = rel(out[r, :T], want), rel(out[r, :T], alone)
        print(f"hubert[{layers} layers] row {r} ({len(w)} samples, {T} frames): rel-L2 vs oracle {e_oracle:.2e}, vs the row alone {e_alone:.2e}")
        assert e_oracle <= TOL_NET, (r, e_oracle)


def test_normalize_kernel_bit_exact(ops):
    from easevoice_trainer_b200 import normalize_ssl as ns
    rng = np.random.default_rng(3)
    rows = [rng.standard_normal(5000).astype(np.float32) * 0.2, rng.standard_normal(3001).astype(np.float32),
            (rng.standard_normal(4000) / 2).astype(np.float32), np.zeros(2000, np.float32), rng.standard_normal(4100).astype(np.float32)]
    rows[1] *= np.float32(1.9) / np.abs(rows[1]).max()                          # wraps in int16
    rows[4] *= np.float32(0.9) / np.abs(rows[4]).max()
    rows[2][17] = 2.2000000476837                                              # float32(2.2) > 2.2 in float64: skipped
    nan_row = rows[0].copy()
    nan_row[100] = np.nan
    inf_row = rows[0][:1000].copy()
    inf_row[5] = np.inf
    rows += [nan_row, inf_row]
    L = max(len(r) for r in rows)
    x = np.zeros((len(rows), L), np.float32)
    for r, a in enumerate(rows):
        x[r, :len(a)] = a
    a32, a32b, status = ops.ssl_normalize(torch.from_numpy(x).to(DEV), torch.tensor([len(a) for a in rows], dtype=torch.int32, device=DEV))
    a32, a32b, status = a32.cpu().numpy(), a32b.cpu().numpy(), status.cpu().tolist()
    code = {ssl_oracle.OK: ns.SSL_OK, ssl_oracle.SKIP: ns.SSL_SKIP, ssl_oracle.NONFINITE: ns.SSL_NONFINITE}
    assert status == [ns.SSL_OK, ns.SSL_OK, ns.SSL_SKIP, ns.SSL_NONFINITE, ns.SSL_OK, ns.SSL_NONFINITE, ns.SSL_SKIP]
    for r, a in enumerate(rows):
        st, w32, wb = ssl_oracle.normalize(a)
        assert status[r] == code[st], r
        assert (a32[r, len(a):] == 0).all() and (a32b[r, len(a):] == 0).all()
        if st == ssl_oracle.OK:
            assert np.array_equal(a32[r, :len(a)], ssl_oracle.to_int16(w32)), r
            assert np.array_equal(a32b[r, :len(a)].view(np.int32), wb.view(np.int32)), r
        elif st == ssl_oracle.NONFINITE:
            assert np.isnan(a32b[r, :len(a)]).all()
    assert (np.abs(ssl_oracle.normalize(rows[1])[1]) > 32767).any()


def test_resampler_taps_against_float64(ops):
    from easevoice_trainer_b200 import normalize_ssl as ns
    rng = np.random.default_rng(4)
    lens = [4001, 4000, 1]
    x = np.zeros((3, 4001), np.float32)
    for r, n in enumerate(lens):
        x[r, :n] = rng.standard_normal(n) * 500
    taps = torch.from_numpy(ns.resample_taps()[1]).to(DEV)
    y = ops.resample_poly(torch.from_numpy(x).to(DEV), taps, 1, 2, 64, 2001).cpu().numpy()
    for r, n in enumerate(lens):
        want = ssl_oracle.resample(x[r, :n].astype(np.float64))
        got = y[r, :n // 2]
        assert rel(got, want[:n // 2]) <= 1e-6 if n > 1 else got.size == 0


def test_write_hubert_features_end_to_end(ops, tmp_path):
    from easevoice_trainer_b200 import normalize_ssl as ns
    net, _, _ = _net(GOLD["layers"], GOLD["param_seed"])
    wav_dir, hub, w32 = tmp_path / "denoised", tmp_path / "4-cnhubert", tmp_path / "5-wav32k"
    for d in (wav_dir, hub, w32):
        os.makedirs(d)
    lines = []
    for c in GOLD["clips"]:
        wavfile.write(wav_dir / c["name"], 32000, ssl_oracle.clip(c))                        # float32 WAV
        lines.append(f"/some/where/{c['name']}|zh|text")
    (tmp_path / "list").write_text("\n".join(lines) + "\n", encoding="utf8")

    def load_audio(path, sr):
        r, a = wavfile.read(path)
        assert r == sr and a.dtype == np.float32
        return a

    args = (tmp_path / "list", wav_dir, hub, w32, net, load_audio)
    failed = ns.write_hubert_features(*args, max_batch=3)
    assert failed == GOLD["failed"]
    for c in GOLD["clips"]:
        n = c["name"]
        if n not in GOLD["written"]:
            assert not (hub / (n + ".pt")).exists() and not (w32 / n).exists(), n
            continue
        sr, wav = wavfile.read(w32 / n)
        assert sr == 32000 and wav.dtype == np.int16 and np.array_equal(wav, GOLD["wav"][n].numpy()), n
        f = torch.load(hub / (n + ".pt"), weights_only=False)
        want = GOLD["ssl"][n]
        assert f.dtype == torch.float32 and f.device.type == "cpu" and f.shape == want.shape and f.shape[:2] == (1, 768)
        assert rel(f, want.detach()) <= TOL_NET, n
    stamps = {p: os.stat(p).st_mtime_ns for d in (hub, w32) for p in (d / q for q in os.listdir(d))}
    assert ns.write_hubert_features(*args) == GOLD["failed"]                  # the failed file is tried again, as the reference does
    assert {p: os.stat(p).st_mtime_ns for d in (hub, w32) for p in (d / q for q in os.listdir(d))} == stamps
