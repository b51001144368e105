"""CPU tests of the 16-bit compute type of the UVR5 VR, DeEcho / DeReverb and MDX23C nets: set_compute_type's validation,
the conv packs it builds, the folded fp32 layers left as they were, pack_conv_h16's rounding, and the float64 emulation
(tests/uvr5_h16_ref.py) against the oracles run in float64 (unrounded), rounding exactly one conv per packed layer."""
import numpy as np
import pytest
import torch

from oracle import mdx23c_oracle as MO
from oracle import uvr5_echo_oracle as EO
from oracle import uvr5_oracle as VO
from tests import uvr5_h16_ref as R

VR_SMALL = dict(size=33966, n_fft=128, seed=21)
ECHO_SMALL = dict(n_fft=128, nout=16, seed=41)
MDX_SMALL = {"audio": {"n_fft": 2048, "hop_length": 512, "dim_f": 512, "chunk_size": 7680},
             "model": {"num_subbands": 2, "num_scales": 2, "num_channels": 16, "growth": 8, "num_blocks_per_scale": 1,
                       "bottleneck_factor": 2}}


def _vr():
    from easevoice_trainer_b200 import uvr5
    P = VO.init_params(VO.param_spec(VR_SMALL["size"]), VR_SMALL["seed"])
    return uvr5.CascadedASPPNet(VR_SMALL["n_fft"], VR_SMALL["size"]).load_state_dict(P), P


def _echo():
    from easevoice_trainer_b200 import uvr5
    P = EO.init_params(EO.param_spec(ECHO_SMALL["n_fft"], ECHO_SMALL["nout"]), ECHO_SMALL["seed"])
    return uvr5.CascadedNet(ECHO_SMALL["n_fft"], ECHO_SMALL["nout"]).load_state_dict(P), P


def _mdx():
    from easevoice_trainer_b200 import mdx23c
    cfg = MO.config(MDX_SMALL)
    P = MO.init_params(MO.param_spec(cfg), 301)
    return mdx23c.MDX23C(cfg).load_state_dict(P), P, cfg


def _conv_layers(m):
    """-> {key: fp32 conv weight [N, k, k, C]} that the model runs on evk_conv2d_fwd"""
    if hasattr(m, "layers"):
        return {p: L["w"] for p, L in m.layers.items() if "k" in L}
    return {k: v for k, v in m.w.items() if v.dim() == 4 and ".upscale." not in k}


def _snapshot(m):
    tree = m.layers if hasattr(m, "layers") else m.w
    copy = lambda v: v.clone() if torch.is_tensor(v) else v          # noqa: E731
    return {k: ({kk: copy(vv) for kk, vv in v.items()} if isinstance(v, dict) else copy(v)) for k, v in tree.items()}


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return torch.equal(a, b) if torch.is_tensor(a) else a == b


@pytest.mark.parametrize("which", ["vr", "echo", "mdx"])
def test_set_compute_type_validation_and_packs(which):
    from easevoice_trainer_b200 import ops
    m = {"vr": _vr, "echo": _echo, "mdx": _mdx}[which]()[0]
    before = _snapshot(m)
    convs = _conv_layers(m)
    assert m.compute_type is None and m._h16 == {}
    for dt in (torch.float16, torch.bfloat16):
        assert m.set_compute_type(dt) is m and m.compute_type is dt
        W = m._h16_weights()
        assert W.keys() == convs.keys() and W is m._h16_weights()      # built once per compute type
        for k, w in W.items():
            N, kk, _, C = convs[k].shape
            assert isinstance(w, ops.PackedH16) and w.w.dtype == dt and w.K == kk * kk * C
            assert w.w.shape == (N, (w.K + 63) // 64 * 64)
            assert torch.equal(w.w[:, :w.K], convs[k].reshape(N, -1).to(dt)) and not w.w[:, w.K:].any()
    assert set(m._h16) == {"torch.float16", "torch.bfloat16"}
    for bad in (torch.float32, torch.float64, "float16", torch.int8, 16):
        with pytest.raises(ValueError):
            m.set_compute_type(bad)
    assert m.compute_type is torch.bfloat16
    assert m.set_compute_type(None) is m and m.compute_type is None
    assert _same(_snapshot(m), before)                      # the fp32 layers are those of a fresh model
    m.to("cpu")
    assert m._h16 == {}                                     # packs follow the device


def test_from_pretrained_compute_type(tmp_path):
    from easevoice_trainer_b200 import mdx23c, uvr5
    m, P = _vr()
    torch.save(P, tmp_path / "vr.pth")
    _, PE = _echo()
    torch.save(PE, tmp_path / "echo.pth")
    _, PM, cfg = _mdx()
    torch.save(PM, tmp_path / "mdx.ckpt")
    for dt in (None, torch.float16, torch.bfloat16):
        a = uvr5.CascadedASPPNet.from_pretrained(str(tmp_path / "vr.pth"), n_fft=128, device="cpu", compute_type=dt)
        b = uvr5.CascadedNet.from_pretrained(str(tmp_path / "echo.pth"), n_fft=128, device="cpu", compute_type=dt)
        c = mdx23c.MDX23C.from_pretrained(str(tmp_path / "mdx.ckpt"), cfg, device="cpu", compute_type=dt)
        assert a.compute_type is dt and b.compute_type is dt and c.compute_type is dt
        assert _same(a.layers, m.layers)
    with pytest.raises(ValueError):
        uvr5.CascadedNet.from_pretrained(str(tmp_path / "echo.pth"), n_fft=128, device="cpu", compute_type=torch.float32)


def test_pack_conv_h16_rounding():
    from easevoice_trainer_b200 import ops
    one = 1.0
    # fp16: spacing 2^-10 at 1; bf16: 2^-7.  Midpoints go to the even neighbour, points past them away.
    for dt, ulp in ((torch.float16, 2.0 ** -10), (torch.bfloat16, 2.0 ** -7)):
        vals = torch.tensor([one + ulp / 2, one + 3 * ulp / 2, one + ulp / 2 + ulp / 64, -(one + ulp / 2), 1e-3],
                            dtype=torch.float32)
        want = torch.tensor([one, one + 2 * ulp, one + ulp, -one, 1e-3], dtype=torch.float32).to(dt)
        w = torch.zeros(3, 3, 3, 2)
        w.view(-1)[:5] = vals
        p = ops.pack_conv_h16(w, dt)
        assert p.K == 18 and p.w.shape == (3, 64) and p.w.dtype == dt
        assert torch.equal(p.w.reshape(-1)[:5].view(torch.int16), want.view(torch.int16))
        assert not p.w[:, 18:].any()
    # fp16 overflow is +-inf, as the torch cast makes it
    p = ops.pack_conv_h16(torch.tensor([7e4, -7e4, 65504.0]).reshape(3, 1, 1, 1), torch.float16)
    assert p.w[0, 0] == float("inf") and p.w[1, 0] == float("-inf") and p.w[2, 0] == 65504
    # an fp16 checkpoint keeps its bits through the fp32 layers
    g = torch.Generator().manual_seed(0)
    w16 = (torch.randn(40, 3, 3, 34, generator=g) * 0.1).half()
    p = ops.pack_conv_h16(w16.float(), torch.float16)
    assert torch.equal(p.w[:, :306].view(torch.int16), w16.reshape(40, -1).view(torch.int16))
    with pytest.raises(ValueError):
        ops.pack_conv_h16(w16.float(), torch.float32)


class _Count:
    """counts the conv2d calls _RoundedConvF rounds"""

    def __init__(self, monkeypatch):
        self.n = 0
        orig = R._RoundedConvF.conv2d

        def conv2d(obj, x, w, *args, **kw):
            groups = kw.get("groups", args[4] if len(args) > 4 else 1)
            if groups == 1 and not any(w is k for k in obj.keep):
                self.n += 1
            return orig(obj, x, w, *args, **kw)
        monkeypatch.setattr(R._RoundedConvF, "conv2d", conv2d)


def _vr_input(n_fft, seed, B=1):
    bins = n_fft // 2 + 1
    x = torch.from_numpy(np.abs(VO.make_spec(seed, bins, 512 * B))).reshape(2, bins, B, 512).permute(2, 0, 1, 3)
    return (x / x.max()).contiguous()


def test_emulation_vr(monkeypatch):
    m, P = _vr()
    x = _vr_input(128, 7)
    agg = {"value": 0.1, "split_bin": 20, "aggr_correction": None}
    P64 = {k: (v.double() if v.is_floating_point() else v) for k, v in P.items()}
    ref = VO.predict(P64, x.double(), agg, 128, True)
    assert torch.equal(R.vr_predict(P, x, agg, None, 128, True), ref)
    cnt = _Count(monkeypatch)
    h = R.vr_predict(P, x, agg, torch.float16, 128, True)
    assert cnt.n == len(_conv_layers(m))                   # one rounded conv per packed layer, the mask head unrounded
    e = float((h - ref).norm() / ref.norm())
    assert 0 < e < 1e-2, e


def test_emulation_echo(monkeypatch):
    m, P = _echo()
    x = _vr_input(128, 8)
    P64 = {k: (v.double() if v.is_floating_point() else v) for k, v in P.items()}
    with torch.no_grad():
        ref = EO.predict(P64, x.double(), None, 128, EO.lstm_modules(P64, "cpu", torch.float64))
    assert torch.equal(R.echo_predict(P, x, None, 128), ref)
    cnt = _Count(monkeypatch)
    h = R.echo_predict(P, x, torch.bfloat16, 128)
    assert cnt.n == len(_conv_layers(m))
    e = float((h - ref).norm() / ref.norm())
    assert 0 < e < 5e-2, e


def test_emulation_inference_matches_the_oracle_window_loop():
    _, P = _vr()
    spec = VO.make_spec(3, 65, 300)
    data = {"window_size": 512, "tta": True}
    P64 = {k: (v.double() if v.is_floating_point() else v) for k, v in P.items()}
    got = R.inference(lambda w: R.vr_predict(P, w, None, None, 128, True), spec, data, VO.OFFSET, "cpu")
    ref = VO.inference(P64, spec.astype(np.complex128), None, data, 128, True)[0]
    assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()     # only the fp32 normalisation differs


def test_emulation_mdx(monkeypatch):
    m, P, cfg = _mdx()
    raw = MO.make_audio(302, (2, 2, 7680))
    P64 = {k: v.double() for k, v in P.items()}
    ref = MO.forward(P64, cfg, raw.double())
    assert torch.equal(R.mdx_forward(P, cfg, raw, None), ref)
    cnt = _Count(monkeypatch)
    h = R.mdx_forward(P, cfg, raw, torch.float16)
    assert cnt.n == len(_conv_layers(m))
    e = float((h - ref).norm() / ref.norm())
    assert 0 < e < 1e-2, e
