"""Every output of the stage-2 attention operator (ops.attention: the TextEncoder's windowed self-attention, the
MelStyleEncoder's and the MRTE cross attention) against float64, element for element, in TF32 and in 3xTF32 mode.

tests/s2_attention_ref.py states the operands, the error model and the case table.  A probe v that is the identity on one
key block per head returns every probability Pd[b][i][j] in one forward, and a probe Ev of unit rows returns the band
Pd[i][i + r - win] tap by tap, so a key wrongly admitted, a band off by one diagonal or a mask the backward drew
differently shows as wrong elements, which a whole-tensor relative-L2 gate averages away.  Each test also asserts, from
the library's dispatch accounting, which kernel family ran each of the five contractions.
"""
import math

import pytest
import torch

from tests import s2_attention_ref as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
WORST, BIAS = {}, {}
OUTPUTS = ("out", "dq", "dk", "dv", "dEk", "dEv")


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    L = lib.init()
    L.evk_set_precise(0)
    try:
        yield ops
    finally:
        L.evk_set_precise(0)
        L.evk_set_backend(1)
        L.evk_set_backend_tma(1)
        for k in sorted(WORST):
            print(f"worst err / gate  {k}: {WORST[k]:.3f}")
        for k in sorted(BIAS):
            print(f"signed mean of (out - ref) / |ref| over |ref| above the median  {k}: {BIAS[k]:+.3e}")


@pytest.fixture(params=list(R.MODES))
def mode(request, ops):
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1 if request.param == "3xtf32" else 0)
    try:
        yield request.param
    finally:
        lib.init().evk_set_precise(0)


def _padded(x, grad):
    """a column slice of a wider buffer whose pitch padding is NaN"""
    B, T, C = x.shape
    buf = torch.full((B, T, C + 4), float("nan"), device=DEV)
    buf[..., :C] = x.float().to(DEV)
    return buf[..., :C].requires_grad_(grad)


def _i32(lens):
    return None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV)


def _run(ops, c, H, q, k, v, Ek, Ev, dout=None):
    """ops.attention on the device -> dict of outputs (and gradients) and the dispatch accounting of each direction"""
    ql, kl = R.case_lens(c)
    grad = dout is not None
    qd, kd, vd = (_padded(t, grad) for t in (q, k, v))
    Ekd = Evd = None
    if c["win"] is not None:
        Ekd, Evd = (t[None].float().to(DEV).requires_grad_(grad) for t in (Ek, Ev))
    ops.dispatch_reset()
    out = ops.attention(qd, kd, vd, heads=H, scale=c["scale"], Ek=Ekd, Ev=Evd, window=c["win"], fill=c["fill"], qlen=_i32(ql),
                        klen=_i32(kl), p_drop=c["p"], tag=R.DROP_TAG)
    got = dict(out=out.detach(), fwd=ops.dispatch_stats())
    if grad:
        ops.dispatch_reset()
        out.backward(dout.float().to(DEV))
        got.update(dq=qd.grad, dk=kd.grad, dv=vd.grad, bwd=ops.dispatch_stats())
        if c["win"] is not None:
            got.update(dEk=Ekd.grad[0], dEv=Evd.grad[0])
    return got


def _ref(c, H, mode, q, k, v, Ek, Ev, dout=None, keep=None, generic=None):
    """float64 reference and model on the device"""
    ql, kl = R.case_lens(c)
    q, k, v, Ek, Ev, dout = (None if t is None else t.to(DEV) for t in (q, k, v, Ek, Ev, dout))
    r = R.attention_f64(q, k, v, Ek, Ev, H, c["win"], c["scale"], c["fill"], ql, kl, keep=keep, p=c["p"], dout=dout)
    return r, R.model(r, q, k, v, Ek, Ev, H, c["win"], c["scale"], mode, dout=dout, p=c["p"], generic=generic)


def _check(c, what, got, ref, bound, mode, family, keys=None):
    text = R.report(c, what, got, ref, bound, keys)
    if text:
        pytest.fail(f"{mode}: {text}")
    w = R.worst(got, ref, bound)
    key = f"{what:14s} {mode:6s} P.V on {family}"
    WORST[key] = max(WORST.get(key, 0.0), w)
    return w


def _family(c, mode):
    return c["families"]["pv"] if mode == "tf32" else "fwd_mma_sync"


def _assert_families(ops, c, H, mode, got):
    """each product is 2 Z Tq Tk dk flops; the accounting must put exactly the expected multiple on each slot"""
    F = 2.0 * c["B"] * H * c["Tq"] * c["Tk"] * (c["C"] // c["H"])
    fam = {n: (f if mode == "tf32" or f.startswith("wgrad") else "fwd_mma_sync") for n, f in c["families"].items()}
    for stats, names in ((got["fwd"], ("qk", "pv")), (got.get("bwd"), ("dov", "dsk", "dv", "dk"))):
        if stats is None:
            continue
        want = dict.fromkeys(ops.DISPATCH_SLOTS, 0.0)
        for n in names:
            want[fam[n]] += F
        assert stats == pytest.approx(want, rel=1e-12), (c["name"], mode, names, stats)


def _readouts(ops, c, mode, keep_fn=None):
    """the probability readout and, with a window, the band readout; keep_fn(H') -> bool [B, H', Tq, Tk] under dropout"""
    q, k, V, keys, Ek = R.readout_inputs(c, 11)
    Hr = R.readout_heads(c)
    dk = c["C"] // c["H"]
    fam = _family(c, mode)
    keep = None if keep_fn is None else keep_fn(Hr)
    Ev0 = None if c["win"] is None else torch.zeros(2 * c["win"] + 1, dk, dtype=torch.float64)
    r, m = _ref(c, Hr, mode, q, k, V, Ek, Ev0, keep=keep)
    got = _run(ops, c, Hr, q, k, V, Ek, Ev0)["out"]
    ws = [_check(c, "readout", got, r["out"], m["out"], mode, fam, keys)]
    want_zero = (R.gather_keys(r["Pd"], keys) == 0).cpu()
    assert torch.equal(got.cpu() == 0, want_zero), f"{c['name']} {mode}: the zero set is not the masked-or-dropped set"
    if keep is None:                                                      # every row of probabilities sums to 1
        rs, rb = got.double().sum(-1).cpu(), m["out"].sum(-1).cpu()
        assert bool(((rs - 1).abs() <= R.SAFETY * rb + R.U32 * c["Tk"]).all()), (c["name"], float((rs - 1).abs().max()))
    if c["win"] is not None:
        probe = R.band_probe(c["win"], dk)
        rb_, mb = _ref(c, Hr, mode, q, k, torch.zeros_like(V), Ek, probe, keep=keep)
        gb = _run(ops, c, Hr, q, k, torch.zeros_like(V), Ek, probe)["out"]
        ws.append(_check(c, "band readout", gb, rb_["out"], mb["out"], mode, fam))
        W = 2 * c["win"] + 1
        outside = ~R.band_index(c["Tq"], c["Tk"], c["win"], "cpu")[1]
        assert bool((R.heads(gb, Hr)[..., :W].cpu()[:, :, outside] == 0).all()), f"{c['name']} {mode}: a band tap outside [0, Tk) is not zero"
    return ws


@pytest.mark.parametrize("c", R.CASES, ids=lambda c: c["name"])
def test_probability_readout(ops, mode, c):
    ws = _readouts(ops, c, mode)
    print(f"{c['name']} {mode}: worst err / gate readout " + " ".join(f"{w:.3f}" for w in ws))


def _forward_backward(ops, c, mode, keep=None):
    q, k, v, do, Ek, Ev = R.case_inputs(c, 1)
    r, m = _ref(c, c["H"], mode, q, k, v, Ek, Ev, dout=do, keep=keep)
    got = _run(ops, c, c["H"], q, k, v, Ek, Ev, dout=do)
    names = [n for n in OUTPUTS if n in m]
    ws = {n: _check(c, n, got[n], r[n], m[n], mode, _family(c, mode)) for n in names}
    _assert_families(ops, c, c["H"], mode, got)
    print(f"{c['name']} {mode}: worst err / gate " + " ".join(f"{n} {w:.3f}" for n, w in ws.items()))


@pytest.mark.parametrize("c", R.CASES, ids=lambda c: c["name"])
def test_forward_backward(ops, mode, c):
    _forward_backward(ops, c, mode)


@pytest.mark.parametrize("c", R.DROP_CASES, ids=lambda c: c["name"])
def test_dropout(ops, mode, c):
    ops.manual_seed(R.DROP_SEED, DEV)
    seed, offset = ops.rng_state(DEV).cpu().tolist()
    sid = ops.stream_id(R.DROP_TAG)
    ld = (c["Tk"] + 3) // 4 * 4

    def keep_fn(H):
        km = R.keep_mask(seed, offset, sid, (c["B"] * H, c["Tq"], ld), c["p"])
        return km.view(c["B"], H, c["Tq"], ld)[..., :c["Tk"]].to(DEV)
    ws = _readouts(ops, c, mode, keep_fn)
    keep = keep_fn(c["H"])
    drop = 1.0 - float(keep.double().mean())
    assert abs(drop - c["p"]) <= 3 * math.sqrt(c["p"] * (1 - c["p"]) / keep.numel()), drop
    _forward_backward(ops, c, mode, keep)                                # gradients under the mask the forward drew
    assert ops.rng_state(DEV).cpu().tolist() == [seed, offset]
    print(f"{c['name']} {mode}: worst err / gate readout " + " ".join(f"{w:.3f}" for w in ws) + f", drop fraction {drop:.4f}")


@pytest.mark.parametrize("c", R.GENERIC_CASES, ids=lambda c: c["name"])
def test_generic_operands(ops, mode, c):
    """normal q, k, v: K and V enter gconv_tc_kernel as raw fp32 bits (truncated), the mma.sync kernel rounds them"""
    q, k, v, _, Ek, Ev = R.case_inputs(c, 2, generic=True)
    q, k, v = (t.float().double() for t in (q, k, v))
    fam = _family(c, mode)
    r, m = _ref(c, c["H"], mode, q, k, v, Ek, Ev, generic=fam)
    got = _run(ops, c, c["H"], q, k, v, Ek, Ev)
    w = _check(c, "generic out", got["out"], r["out"], m["out"], mode, fam)
    _assert_families(ops, c, c["H"], mode, got)
    ref = r["out"].cpu()
    big = ref.abs() > ref.abs().median()
    BIAS[f"{c['name']} {mode} ({fam})"] = float(((got["out"].double().cpu() - ref) / ref.abs())[big].mean())
    print(f"{c['name']} {mode} ({fam}): worst err / gate out {w:.3f}")
