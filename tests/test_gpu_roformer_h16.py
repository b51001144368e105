"""GPU tests of the Roformers' float16 / bfloat16 compute type (`pytest -m gpu`): evk_rope_attn_fwd_h16 against the float64
emulation of its contract at both axis layouts, the 16-bit Linear on the mono band-split operand (column slices at 8-byte
offsets), BSRoformer / MelBandRoformer.forward and bs_roformer.demix_track against the float64 emulation of the whole 16-bit
network (tests/roformer_h16_ref.py), chunk and launch invariance, and switching between compute types.

Measured on one H100 80GB HBM3 at 700 W (rel-L2 against the emulation):
  evk_rope_attn_fwd_h16 over the grid below: fp16 at most 1.0e-4, bf16 at most 7.8e-4 (both at L >= 801).
  forward / demix_track over the five configurations: fp16 at most 7.5e-4, bf16 at most 6.1e-3 (Mel-Band default).
  Against the fp32 reference's goldens (printed, not gated): fp16 at most 1.3e-3, bf16 at most 8.6e-3.
The gates are the TF32 kernel's and network's (2e-3, 3e-3) for fp16, and 8x that for bf16, whose unit roundoff is 8x fp16's."""
import os

import numpy as np
import pytest
import torch

from oracle import bs_roformer_oracle as BO
from oracle import mel_roformer_oracle as MO
from tests import roformer_h16_ref as RH

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
TYPES = [torch.float16, torch.bfloat16]
TOL_ATTN = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}
TOL_NET = {torch.float16: 3e-3, torch.bfloat16: 2e-2}
GOLD = {False: torch.load(os.path.join(ROOT, "tests", "golden", "bs_roformer.pt"), weights_only=False),
        True: torch.load(os.path.join(ROOT, "tests", "golden", "mel_roformer.pt"), weights_only=False)}
NETS = [(False, "small"), (False, "full"), (True, "small"), (True, "default"), (True, "mono")]


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


def _set_precise(on):
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1 if on else 0)


def rel(a, b):
    a, b = (torch.as_tensor(np.asarray(t)) if not torch.is_tensor(t) else t for t in (a, b))
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---- the attention kernel ---------------------------------------------------------------------------------------------
def _geo(layout, X):
    B, T, Fb, _ = X.shape
    return (B, T * Fb, Fb, 1, Fb) if layout == "time" else (B * T, Fb, 1, 0, 1)


def _run_attn(ops, X, H, L, layout, dtype, extra=4):
    D = H * 64
    out = torch.full((X.shape[0] * X.shape[1] * X.shape[2], D + extra), 7.0, device=DEV)
    ops.rope_attn_h16(X.view(-1, X.shape[-1]), RH.cos_sin(L, DEV).float(), out[:, :D], H, L, *_geo(layout, X), dtype)
    return out


def _attn_emulated(X, H, L, layout, dtype):
    """the kernel's contract in float64 -> [B, T, F, H*64]"""
    D = H * 64
    Xs = (X.permute(0, 2, 1, 3) if layout == "time" else X).double()
    n = Xs.shape[0] * Xs.shape[1]
    Xs = Xs.reshape(n, L, -1)
    o = RH.attention(RH.rounding(dtype), Xs[..., :3 * D], Xs[..., 3 * D:3 * D + H], H, RH.cos_sin(L, X.device))
    if layout == "time":
        return o.reshape(X.shape[0], X.shape[2], L, D).permute(0, 2, 1, 3)
    return o.reshape(X.shape[0], X.shape[1], L, D)


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("H", [2, 8])
@pytest.mark.parametrize("L", [1, 7, 62, 801, 1500])
@pytest.mark.parametrize("layout", ["time", "freq"])
def test_rope_attn_h16_vs_float64(ops, layout, L, H, dtype):
    g = torch.Generator().manual_seed(L * 10 + H)
    D = H * 64
    ld = (3 * D + H + 3) // 4 * 4 + 4
    shape = (2, L, 3, ld) if layout == "time" else (1, 3, L, ld)
    X = (torch.randn(shape, generator=g) * 1.5).to(DEV)
    out = _run_attn(ops, X, H, L, layout, dtype)
    assert torch.equal(out, _run_attn(ops, X, H, L, layout, dtype))       # bit-reproducible
    assert (out[:, D:] == 7).all()                                          # nothing outside the output slice is written
    _set_precise(True)
    try:
        assert torch.equal(out, _run_attn(ops, X, H, L, layout, dtype))   # evk_set_precise has no effect
    finally:
        _set_precise(False)
    # a sequence's bits do not depend on how many sequences share the launch
    one = _run_attn(ops, (X[:1] if layout == "time" else X[:, :1]).contiguous(), H, L, layout, dtype)
    assert torch.equal(one, out[:one.shape[0]])
    e = rel(out[:, :D], _attn_emulated(X, H, L, layout, dtype).reshape(-1, D))
    print(f"rope_attn_h16 {layout} L={L} H={H} {dtype} rel-L2 {e:.3g}")
    assert e <= TOL_ATTN[dtype], e


def test_rope_attn_h16_rejects_other_types(ops):
    X = torch.zeros(1, 4, 1, 3 * 128 + 4, device=DEV)
    with pytest.raises(ValueError):
        _run_attn(ops, X, 2, 4, "time", torch.float32)


# ---- the 16-bit Linear on the mono band-split operand -----------------------------------------------------------------
@pytest.mark.parametrize("dtype", TYPES)
def test_linear_h16_on_column_slices_at_8_byte_offsets(ops, dtype):
    """a mono model's band i reads columns [2 off[i], 2 off[i+1]) of the band-split operand: 8-byte, not 16-byte, offsets"""
    g = torch.Generator().manual_seed(3)
    rows, N = 300, 96
    xb = torch.randn(rows, 2 * 65 + 6, generator=g).to(DEV)
    for c0, C in ((2, 4), (6, 14), (10, 2 * 59)):
        w = torch.randn(N, C, generator=g) / C ** 0.5
        b = 0.1 * torch.randn(N, generator=g)
        y = torch.full((rows, N + 4), 7.0, device=DEV)
        ops.linear_h16(xb[:, c0:c0 + C], ops.pack_weight_h16(w.to(DEV), dtype), bias=b.to(DEV), out=y[:, :N])
        assert (y[:, N:] == 7).all()
        h = RH.rounding(dtype)
        ref = h(xb[:, c0:c0 + C].cpu().double()) @ h(w.double()).T + b.double()
        e = rel(y[:, :N], ref)
        assert e <= 1e-6, (c0, C, e)                                        # products exact, fp32 sums of <= 118 terms


# ---- the networks -----------------------------------------------------------------------------------------------------
def _net(mel, name, dtype):
    from easevoice_trainer_b200 import bs_roformer, mel_band_roformer
    O = MO if mel else BO
    case = GOLD[mel][name]
    cfg = dict(O.DEFAULT if mel else O.SHIPPED)
    cfg.update(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    cls = mel_band_roformer.MelBandRoformer if mel else bs_roformer.BSRoformer
    return O, case, cfg, P, cls(**cfg).to(DEV).load_state_dict(P).set_compute_type(dtype)


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("mel,name", NETS)
def test_forward_vs_emulation(mel, name, dtype):
    O, case, cfg, P, m = _net(mel, name, dtype)
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    out = m.forward(raw)
    emu = RH.forward(P, cfg, raw, dtype, mel=mel)
    assert out.shape == emu.shape
    e = rel(out, emu)
    g = rel(out[..., ::case["stride"]], case["forward"])
    print(f"forward {'mel' if mel else 'bs'} {name} {dtype} rel-L2 {e:.3g} vs emulation, {g:.3g} vs fp32 golden")
    assert e <= TOL_NET[dtype], e


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("mel,name", NETS)
def test_demix_vs_emulation(mel, name, dtype):
    from easevoice_trainer_b200 import bs_roformer
    O, case, cfg, P, m = _net(mel, name, dtype)
    mix = O.make_audio(case["audio_seed"] + 100, (2 if cfg["stereo"] else 1, int(case["demix_chunks"] * O.CHUNK)))
    got = bs_roformer.demix_track(m, mix, DEV)["vocals"]
    emu = RH.demix_track(P, cfg, mix, dtype, mel=mel, device=DEV)["vocals"]
    e = rel(got, emu)
    g = rel(got[:, case["demix_idx"].numpy()], case["demix"])
    print(f"demix {'mel' if mel else 'bs'} {name} {dtype} rel-L2 {e:.3g} vs emulation, {g:.3g} vs fp32 golden")
    assert e <= TOL_NET[dtype], e
    assert np.array_equal(np.nonzero((got == 0).all(0))[0], case["demix_zero"].numpy())


@pytest.mark.parametrize("dtype", TYPES)
def test_chunk_independent_of_its_launch_and_max_chunks(dtype):
    from easevoice_trainer_b200 import bs_roformer
    O, case, cfg, P, m = _net(False, "small", dtype)
    a = O.make_audio(5, (4, 2, 44100)).to(DEV)
    both = m.forward(a)
    assert torch.equal(both[2:3], m.forward(a[2:3].contiguous()))
    mix = O.make_audio(case["audio_seed"] + 100, (2, int(case["demix_chunks"] * O.CHUNK)))
    x1 = bs_roformer.demix_track(m, mix, DEV, max_chunks=1)["vocals"]
    x4 = bs_roformer.demix_track(m, mix, DEV, max_chunks=4)["vocals"]
    assert np.array_equal(x1, x4)


@pytest.mark.parametrize("mel,name", [(False, "small"), (True, "mono")])
def test_switching_compute_types(mel, name):
    O, case, cfg, P, m = _net(mel, name, None)
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    fresh = m.forward(raw)
    _, _, _, _, h = _net(mel, name, torch.float16)
    y16 = h.forward(raw)
    assert all(k[0] is None for k in h._packed)                            # a 16-bit model builds no TF32 packs
    _set_precise(True)
    try:
        assert torch.equal(h.forward(raw), y16)                            # the precise mode leaves 16-bit outputs as they are
    finally:
        _set_precise(False)
    assert not torch.equal(y16, fresh)
    assert torch.equal(h.set_compute_type(None).forward(raw), fresh)       # fp16 -> None: the TF32 bits of a fresh model
    assert torch.equal(h.set_compute_type(torch.float16).forward(raw), y16)
    assert torch.equal(m.set_compute_type(torch.float16).forward(raw), y16)
