"""CPU tests of the Roformers' 16-bit compute type: set_compute_type's validation, the packed-weight key following it and
the packs it builds, the folded host weights left as they were, and the float64 emulation (tests/roformer_h16_ref.py)
against the fp32 oracles run in float64 (unrounded) and against a direct per-sequence computation of the attention."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import bs_roformer_oracle as BO
from oracle import mel_roformer_oracle as MO
from tests import roformer_h16_ref as R

BS_TINY = dict(BO.SHIPPED, dim=32, depth=1, heads=2, stft_n_fft=256, stft_win_length=256, stft_hop_length=64,
               freqs_per_bands=(16, 48, 65))
MEL_TINY = dict(MO.DEFAULT, dim=32, depth=2, heads=1, num_bands=8, stft_n_fft=256, stft_win_length=256, stft_hop_length=64,
                stereo=False, mask_estimator_depth=1, match_input_audio_length=True)


class _Lib:
    """lib.init() stand-in for the TF32 key: only the precise mode is read"""
    def __init__(self):
        self.precise = 0

    def evk_get_precise(self):
        return self.precise


def test_set_compute_type_validation_and_packs(monkeypatch):
    from easevoice_trainer_b200 import bs_roformer, ops
    stub = _Lib()
    monkeypatch.setattr(bs_roformer.lib, "init", lambda: stub)
    m = bs_roformer.BSRoformer(**BS_TINY).load_state_dict(BO.init_params(BO.param_spec(BS_TINY), 3))
    host = {k: v.clone() for k, v in m.host_w.items()}
    bias = {k: v.clone() for k, v in m.bias.items()}
    assert m.compute_type is None and m._weights_key() == (0, "None")
    stub.precise = 1
    assert m._weights_key() == (1, "None")
    for dt in (torch.float16, torch.bfloat16):
        assert m.set_compute_type(dt) is m and m.compute_type is dt
        assert m._weights_key() == (None, str(dt))              # the precise mode does not select a 16-bit pack
        W = m._weights()
        assert W.keys() == host.keys()
        for k, w in W.items():
            assert isinstance(w, ops.PackedH16) and w.w.dtype == dt and w.K == host[k].shape[1]
            assert torch.equal(w.w[:, :w.K], host[k].to(dt)) and not w.w[:, w.K:].any()
    assert set(m._packed) == {(None, "torch.float16"), (None, "torch.bfloat16")}   # no TF32 pack was built
    for bad in (torch.float32, "float16", torch.int8, 16):
        with pytest.raises(ValueError):
            m.set_compute_type(bad)
    assert m.compute_type is torch.bfloat16
    assert m.set_compute_type(None) is m and m._weights_key() == (1, "None")
    assert all(torch.equal(m.host_w[k], v) for k, v in host.items()) and m.host_w.keys() == host.keys()
    assert all(torch.equal(m.bias[k], v) for k, v in bias.items()) and m.bias.keys() == bias.keys()


def test_from_pretrained_compute_type(tmp_path):
    from easevoice_trainer_b200 import bs_roformer, mel_band_roformer
    P = BO.init_params(BO.param_spec(BO.SHIPPED), 4)
    torch.save(P, tmp_path / "bs.ckpt")
    assert bs_roformer.BSRoformer.from_pretrained(str(tmp_path / "bs.ckpt"), "cpu").compute_type is None
    m = bs_roformer.BSRoformer.from_pretrained(str(tmp_path / "bs.ckpt"), "cpu", compute_type=torch.float16)
    assert m.compute_type is torch.float16
    cfg = dict(MO.DEFAULT, dim=32, depth=1, heads=1)
    torch.save(MO.init_params(MO.param_spec(cfg), 5), tmp_path / "mel.ckpt")
    m = mel_band_roformer.MelBandRoformer.from_pretrained(str(tmp_path / "mel.ckpt"), "cpu", compute_type=torch.bfloat16)
    assert m.compute_type is torch.bfloat16 and m.dim == 32
    with pytest.raises(ValueError):
        bs_roformer.BSRoformer.from_pretrained(str(tmp_path / "bs.ckpt"), "cpu", compute_type=torch.float64)


@pytest.mark.parametrize("mel", [False, True])
def test_unrounded_emulation_equals_oracle(mel):
    """with h the identity the emulation is the oracle's computation (gamma folding included), in float64"""
    O, cfg = (MO, MEL_TINY) if mel else (BO, BS_TINY)
    S = 2 if cfg["stereo"] else 1
    P = O.init_params(O.param_spec(cfg), 11)
    raw = O.make_audio(12, (2, S, 3001))
    got = R.forward(P, cfg, raw, None, mel=mel)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                  # the oracle in float64: its window and parameters follow
    try:
        ref = O.forward({k: v.double() for k, v in P.items()}, cfg, raw.double())
    finally:
        torch.set_default_dtype(prev)
    assert got.shape == ref.shape and ref.dtype == torch.float64
    e = float((got - ref).norm() / ref.norm())
    assert e <= 1e-12, e


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_attention_emulation_equals_direct_computation(dtype):
    g = torch.Generator().manual_seed(7)
    n, L, H = 3, 37, 2
    qkv, gates = torch.randn(n, L, 3 * H * 64, generator=g, dtype=torch.float64) * 1.5, torch.randn(n, L, H, generator=g).double()
    cs = R.cos_sin(L, "cpu")
    h = R.rounding(dtype)
    got = R.attention(h, qkv, gates, H, cs, block=2)
    want = torch.empty_like(got)
    for u in range(n):
        for hh in range(H):
            q, k, v = (qkv[u, :, (i * H + hh) * 64:(i * H + hh + 1) * 64] for i in range(3))
            for p in range(L):
                qr = h(R.rotate(q[p:p + 1], cs[p:p + 1]))[0]
                s = torch.stack([qr @ h(R.rotate(k[j:j + 1], cs[j:j + 1]))[0] for j in range(L)]) / 8.0
                e = torch.exp(s - s.max())
                want[u, p, hh * 64:(hh + 1) * 64] = (h(e) @ h(v)) / e.sum() / (1.0 + math.exp(-float(gates[u, p, hh])))
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-13)
    # the rounding points matter: unrounded, the result moves by about the unit roundoff
    assert not torch.allclose(got, R.attention(R.rounding(None), qkv, gates, H, cs), rtol=1e-6, atol=0)


def test_folded_linear_is_the_norm_then_the_linear():
    g = torch.Generator().manual_seed(8)
    x, w, b, gamma = (torch.randn(5, 24, generator=g).double(), torch.randn(7, 24, generator=g).double(),
                      torch.randn(7, generator=g).double(), 0.5 + torch.rand(24, generator=g).double())
    ref = F.linear(F.normalize(x, dim=-1) * math.sqrt(24) * gamma, w, b)
    assert torch.allclose(R.lin(R.rounding(None), x, w, b, gamma), ref, rtol=1e-13, atol=1e-13)
