"""CPU rehearsal of tests/test_gpu_s2_attention_elementwise.py: the float64 reference of the stage-2 attention operator
agrees with the oracle's skew-free restatement of attentions.py, an fp32 emulation of the operator stays within the
first-order error model (half the gate) at every element of every case, and the element-wise gate rejects every modelled
kernel fault at the element it touches -- while the whole-tensor relative-L2 gate of checks.check_attention (TOL_TC) lets
the ones that touch few elements through."""
import math

import numpy as np
import pytest
import torch

from oracle import s2_oracle
from tests import attention_ref as A
from tests import exact_ref
from tests import s2_attention_ref as R
from tests.checks import TOL_TC

MODES = tuple(R.MODES)
OUTPUTS = ("out", "dq", "dk", "dv", "dEk", "dEv")
ALL_CASES = R.CASES + R.DROP_CASES


def _keep(c, seed=R.DROP_SEED, sid=3):
    if not c["p"]:
        return None
    Z, ld = c["B"] * c["H"], (c["Tk"] + 3) // 4 * 4
    return R.keep_mask(seed, 0, sid, (Z, c["Tq"], ld), c["p"]).view(c["B"], c["H"], c["Tq"], ld)[..., :c["Tk"]]


def _args(c):
    ql, kl = R.case_lens(c)
    return dict(H=c["H"], win=c["win"], scale=c["scale"], fill=c["fill"], qlen=ql, klen=kl)


def _ref(c, mode, seed=1):
    q, k, v, do, Ek, Ev = R.case_inputs(c, seed)
    keep = _keep(c)
    r = R.attention_f64(q, k, v, Ek, Ev, keep=keep, p=c["p"], dout=do, **_args(c))
    m = R.model(r, q, k, v, Ek, Ev, c["H"], c["win"], c["scale"], mode, dout=do, p=c["p"])
    return (q, k, v, do, Ek, Ev), keep, r, m


# ---- the reference ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [c for c in R.CASES if c["fill"] == -1e4], ids=lambda c: c["name"])
def test_reference_matches_oracle(c):
    """attention_f64 against s2_oracle.relpos_attention (pinned to attentions.py), output and all gradients, with a
    non-zero upstream gradient on dead query rows: a filled logit passes none of it on"""
    B, Tq, Tk, C, H, win = (c[n] for n in ("B", "Tq", "Tk", "C", "H", "win"))
    g = torch.Generator().manual_seed(5)
    q, k, do = (torch.randn(B, T, C, generator=g, dtype=torch.float64) for T in (Tq, Tk, Tq))
    Wv = torch.randn(C, C, generator=g, dtype=torch.float64) / math.sqrt(C)
    eye = torch.eye(C, dtype=torch.float64).unsqueeze(-1)
    P = {"a.conv_q.weight": eye, "a.conv_k.weight": eye, "a.conv_v.weight": Wv.unsqueeze(-1), "a.conv_o.weight": eye}
    dk = C // H
    Ek = Ev = None
    if win is not None:
        Ek, Ev = (torch.randn(2 * win + 1, dk, generator=g, dtype=torch.float64) * dk ** -0.5 for _ in range(2))
        P["a.emb_rel_k"], P["a.emb_rel_v"] = Ek[None].clone().requires_grad_(True), Ev[None].clone().requires_grad_(True)
    ql, kl = R.case_lens(c)
    am = R.visible(B, Tq, Tk, ql, kl, "cpu").double()
    x, cc = q.transpose(1, 2).clone().requires_grad_(True), k.transpose(1, 2).clone().requires_grad_(True)
    y = s2_oracle.relpos_attention(P, "a", x, cc, am, H, win)
    y.backward(do.transpose(1, 2))
    v = k @ Wv.t()
    r = R.attention_f64(q, k, v, Ek, Ev, dout=do, **_args(c))
    dkv = r["dk"] + r["dv"] @ Wv                                         # the oracle's k gradient includes the value path
    pairs = [("out", r["out"], y.transpose(1, 2)), ("dq", r["dq"], x.grad.transpose(1, 2)), ("dk + dv Wv", dkv, cc.grad.transpose(1, 2))]
    if win is not None:
        pairs += [("dEk", r["dEk"], P["a.emb_rel_k"].grad[0]), ("dEv", r["dEv"], P["a.emb_rel_v"].grad[0])]
    for name, got, want in pairs:                                         # 2^-24: the reference uses the kernels' fp32 scale
        assert float((got - want).abs().max()) <= 4 * 2.0 ** -24 * float(want.abs().max()) + 1e-14, (c["name"], name)
    if ql is not None:
        dead = torch.arange(Tq)[None, :] >= torch.tensor(ql)[:, None]
        assert bool((r["dq"][dead] == 0).all()) and bool((x.grad.transpose(1, 2)[dead] == 0).all())


def test_keep_mask_is_the_library_draw():
    """keep_mask against the scalar Philox of attention_ref (known-answer tested in test_cpu_dropout_hash.py), on a padded
    pitch, with a non-zero offset"""
    seed, off, sid, p = R.DROP_SEED, 7, 5, 0.1
    shape = (3, 5, 12)
    km = R.keep_mask(seed, off, sid, shape, p).reshape(-1)
    p32 = float(np.float32(p))
    for e in (0, 1, 2, 3, 4, 59, 118, 179):
        w = A.philox(seed, off + e // 4, sid)[e % 4]
        assert bool(km[e]) == ((w >> 8) * 2.0 ** -24 >= p32), e
    big = R.keep_mask(seed, 0, sid, (8, 352, 352), p)
    n = big.numel()
    assert abs(1.0 - float(big.double().mean()) - p32) < 3 * math.sqrt(p * (1 - p) / n)
    assert R.u32_to_unit(0xFFFFFFFF) < 1.0 and R.u32_to_unit(255) == 0.0


def test_exactness_bounds_hold_from_shapes_alone():
    for c in ALL_CASES:
        assert max(R.exact_bounds(c).values()) <= exact_ref.EXACT_BOUND, c["name"]
        assert c["C"] % c["H"] == 0 and (c["C"] // c["H"]) % 4 == 0


def test_case_table_covers_what_it_claims():
    tk = {c["Tk"] for c in R.CASES}
    assert {R.softmax_block(t) for t in tk} == {64, 128, 256} and {63, 64, 127, 128, 255, 256, 257} <= tk
    assert {t % 4 for t in tk} == {0, 1, 2, 3}
    assert {c["families"]["pv"] for c in R.CASES} == {"fwd_gconv_tc", "fwd_mma_sync"}
    assert any(c["fill"] == float("-inf") and c["masks"] == "k" for c in R.CASES)
    assert any(c["win"] is not None and c["Tq"] < c["win"] for c in R.CASES)
    assert {1, 2, 4, 5, 9} <= {c["Tq"] for c in R.CASES if c["win"] == 4}
    assert any(c["B"] * c["Tq"] * c["C"] > R.G1_CAP for c in R.CASES)
    assert any((c["B"] * c["H"] * c["Tq"]) % R.DE_CHUNK and c["Tq"] < R.DE_CHUNK < 2 * c["H"] * c["Tq"] for c in R.CASES)
    for c in R.CASES[:3]:
        ql, kl = R.case_lens(c)
        assert c["Tk"] in kl and 1 in kl and c["Tk"] % 32 == 0 and c["Tq"] % 32 == 0
    assert {c["p"] for c in R.DROP_CASES} == {0.1, 0.5}


# ---- headroom: the emulation stays within the model ----------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c", ALL_CASES, ids=lambda c: c["name"])
def test_emulation_stays_within_the_model(c, mode):
    (q, k, v, do, Ek, Ev), keep, r, m = _ref(c, mode)
    vis_p = r["P"][r["vis"].expand_as(r["P"]) & (r["P"] > 0)]
    assert float(vis_p.min()) >= R.PROB_FLOOR, c["name"]
    e = R.emulate(q, k, v, Ek, Ev, mode=mode, families=c["families"], keep=keep, p=c["p"], dout=do, **_args(c))
    names = ("P", "Pd") + OUTPUTS + (("band",) if c["win"] is not None else ())
    ws = {n: R.worst(e[n], r[n], m[n]) for n in names if n in m}
    print(f"{c['name']} {mode}: worst emulated err / gate " + " ".join(f"{n} {w:.3f}" for n, w in ws.items()))
    assert max(ws.values()) <= 0.5, ws
    assert bool((e["Pd"][r["Pd"] == 0] == 0).all())                      # masked and dropped probabilities are exact zeros


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c", R.GENERIC_CASES, ids=lambda c: c["name"])
def test_emulation_with_generic_operands_stays_within_the_model(c, mode):
    q, k, v, _, Ek, Ev = R.case_inputs(c, 2, generic=True)
    fam = c["families"]["pv"]
    r = R.attention_f64(q, k, v, Ek, Ev, **_args(c))
    m = R.model(r, q, k, v, Ek, Ev, c["H"], c["win"], c["scale"], mode, generic=fam)
    e = R.emulate(q, k, v, Ek, Ev, mode=mode, families=c["families"], **_args(c))
    w = R.worst(e["out"], r["out"], m["out"])
    print(f"{c['name']} {mode} ({fam}): worst emulated err / gate out {w:.3f}")
    assert w <= 0.5


# ---- sensitivity: the element-wise gate rejects every modelled fault -------------------------------------------------------
def test_gate_rejects_every_modelled_fault():
    mode = "tf32"
    c = dict(R.CASES[0], p=0.1)                                           # the self step shape, dropout on
    (q, k, v, do, Ek, Ev), keep, r, m = _ref(c, mode)
    ql, kl = R.case_lens(c)
    kw = dict(mode=mode, families=c["families"], keep=keep, p=c["p"], dout=do, **_args(c))
    good = R.emulate(q, k, v, Ek, Ev, **kw)
    names = ("P", "Pd", "band") + OUTPUTS
    assert all(not bool(R.outside(good[n], r[n], m[n]).any()) for n in names)
    # the elements each fault may touch: (output, predicate on the index); an admitted key renormalises its whole row
    expect = {"key klen admitted": ("P", lambda i: i[2] < ql[i[0]] and i[3] <= kl[i[0]] < c["Tk"]),
              "dead query rows not filled": ("P", lambda i: i[2] >= ql[i[0]]),
              "boundary drelk taps not zeroed": ("dq", lambda i: i[1] < c["win"] or i[1] >= c["Tk"] - c["win"]),
              "backward mask differs in one float4 group": ("dq", lambda i: i[0] == c["B"] - 1 and i[1] == c["Tq"] // 4 and i[2] >= c["C"] // 2)}
    seen = {}
    for fault in R.FAULTS:
        e = R.emulate(q, k, v, Ek, Ev, fault=fault, **kw)
        bad = {n: R.outside(e[n], r[n], m[n]) for n in names}
        l2 = max(A.rel_l2(e[n], r[n]) for n in OUTPUTS)
        seen[fault] = (any(bool(x.any()) for x in bad.values()), l2)
        print(f"fault {fault!r}: element-wise gate {'rejects' if seen[fault][0] else 'PASSES'} "
              f"({', '.join(n for n, x in bad.items() if bool(x.any()))}); worst rel-L2 of an output {l2:.2e} "
              f"({'passes' if l2 <= TOL_TC else 'fails'} TOL_TC)")
        if fault in expect:                                               # ... at the element the fault touches
            n, touched = expect[fault]
            idx = bad[n].nonzero().tolist()
            assert idx and all(touched(i) for i in idx), (fault, idx[:4])
        if fault == "last rel_dE chunk dropped":
            assert bool(bad["dEk"].any()) and not any(bool(bad[n].any()) for n in names if n != "dEk")
            text = R.report(c, "dEk", e["dEk"], r["dEk"], m["dEk"])
            assert "tap r=" in text and f"{-(-c['B'] * c['H'] * c['Tq'] // R.DE_CHUNK)} rel_dE chunks" in text
    assert all(rej for rej, _ in seen.values()), seen
    # a fault that touches a few of many elements is below TOL_TC of every tensor norm; with this case's ragged lengths
    # (one item of length 1, non-zero upstream gradient on dead rows) the others are not, and the lines above say so
    assert seen["backward mask differs in one float4 group"][1] <= TOL_TC, seen
    text = R.report(c, "dq", R.emulate(q, k, v, Ek, Ev, fault="boundary drelk taps not zeroed", **kw)["dq"], r["dq"], m["dq"])
    assert "i=0 (128-row tile 0)" in text and "rel_dE chunk 0" in text and "softmax block 256" in text
