"""CPU rehearsal of tests/train_ref.py: fp32 emulations of the weight-norm packing, ScaledAdam and quantizer kernels'
summation orders stay within the error model (half the gate) at every element; the float64 references agree with
torch._weight_norm and its autograd gradients, with oracle/gpt_oracle.ScaledAdamOracle over the golden schedule and with
oracle/vq_train_oracle; and modelled faults (a clipping median one slot off, a dropped param_max_rms override, the EMA
counting rows past rows_ref) leave the gate on at least one element."""
import json
import os

import pytest
import torch

from oracle import gpt_oracle, vq_train_oracle
from tests import cudacore_ref as R
from tests import train_ref as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(lr=0.01, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=1000, scalar_lr_scale=0.1, eps=1e-8,
           param_min_rms=1e-5, param_max_rms=3.0, scalar_max=10.0, size_update_period=4)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def within_model(got, ref, what, extra=0.0):
    got = got.double()
    bad = ~torch.isfinite(got) | ((got - ref.v).abs() > ref.e + extra)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the model"


def outside(got, ref, what):
    n = int(R.outside_gate(got, ref).sum())
    print(f"fault '{what}': {n} elements outside the gate")
    assert n > 0, f"fault '{what}' stays inside the gate"


# ---- weight norm ------------------------------------------------------------------------------------------------------------
PACK_SHAPES = [(4, 6, 1), (8, 3, 3), (6, 5, 5), (5, 4, 7), (3, 40, 1), (2, 300, 4)]      # n from 6 to 1200 (> 256 * 4)


@pytest.mark.parametrize("shape", PACK_SHAPES, ids=[f"{a}x{b}x{c}" for a, b, c in PACK_SHAPES])
def test_weight_pack_emulation_within_model(shape):
    g0 = _gen(sum(shape))
    v = torch.randn(*shape, generator=g0)
    v[0] *= 1e-3                                                      # a small-norm row
    g = torch.rand(shape[0], generator=g0) + 0.5
    vf = v.reshape(shape[0], -1)
    ref = T.weight_pack(vf, g)
    within_model(T.emulate_weight_pack(vf, g, round_tf32=False), ref, "precise")
    got = T.emulate_weight_pack(vf, g)
    assert bool(((got.view(torch.int32) & 0x1FFF) == 0).all())
    within_model(got, ref, "tf32", T.tf32_gate(ref, 1.0))
    dpa = torch.randn(vf.shape, generator=g0)
    dv, dg = T.emulate_weight_pack_bwd(vf, g, dpa)
    rdv, rdg = T.weight_pack_bwd(vf, g, dpa)
    within_model(dv, rdv, "dv")
    within_model(dg, rdg, "dg")


def test_weight_pack_fault_tf32_dropped():
    v = torch.randn(16, 64, generator=_gen(1))
    ref = T.weight_pack(v, None)                                     # e = 0: the packed value must be v's TF32 rounding
    got = T.emulate_weight_pack(v, None, round_tf32=False)
    assert bool(((got.view(torch.int32) & 0x1FFF) != 0).any()), "no element has low mantissa bits: the TF32 check is blind"


@pytest.mark.parametrize("shape", [(4, 6, 1), (6, 5, 5), (2, 300, 4)])
def test_weight_norm_reference_is_torch_weight_norm(shape):
    g0 = _gen(7)
    v = torch.randn(*shape, generator=g0, dtype=torch.float64, requires_grad=True)
    g = (torch.rand(shape[0], 1, 1, generator=g0, dtype=torch.float64) + 0.5).requires_grad_(True)
    w = torch._weight_norm(v, g, 0)
    ref = T.weight_pack(v.detach().reshape(shape[0], -1), g.detach().reshape(-1))
    assert float((ref.v - w.detach().reshape(shape[0], -1)).abs().max()) <= 1e-14 * float(w.detach().abs().max())
    dpa = torch.randn(*shape, generator=g0, dtype=torch.float64)
    dv, dg = torch.autograd.grad(w, [v, g], dpa)
    rdv, rdg = T.weight_pack_bwd(v.detach().reshape(shape[0], -1), g.detach().reshape(-1), dpa.reshape(shape[0], -1))
    assert float((rdv.v - dv.reshape(shape[0], -1)).abs().max()) <= 1e-13 * float(dv.abs().max())
    assert float((rdg.v - dg.reshape(-1)).abs().max()) <= 1e-13 * float(dg.abs().max())


def test_tf32_rna():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 2 ** -12, 3.0e-39])
    y = T.tf32_rna(x)
    assert y.tolist()[:5] == [1.0, 1.0 + 2 ** -10, 1.0 + 2 * 2 ** -10, -(1.0 + 2 ** -10), 1.0]       # ties away from zero
    r = torch.randn(10000, generator=_gen(2))
    assert bool(((T.tf32_rna(r) - r).abs() <= T.TF32_REL * r.abs()).all())


# ---- ScaledAdam ----------------------------------------------------------------------------------------------------------------
def fresh_state(nt, cfg):
    return dict(step=0, rms=torch.zeros(nt, dtype=torch.float64), sv=torch.zeros(nt, dtype=torch.float64),
                sg=torch.zeros(cfg["size_update_period"], nt, dtype=torch.float64),
                norms=torch.zeros(cfg["clipping_update_period"], dtype=torch.float64), thr=torch.zeros(2, dtype=torch.float64))


def test_sadam_restatement_matches_oracle_on_golden_schedule():
    """the restatement carried in float64 over tests/golden/scaled_adam.json's schedule (the one check_scaled_adam runs)
    agrees with ScaledAdamOracle step by step; the state is carried from step to step as plain float64 values"""
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "scaled_adam.json")))
    g0 = _gen(gold["seed"])
    shapes = [tuple(s) for s in gold["shapes"]]
    init = [(torch.randn(s, generator=g0) * sc).double() for s, sc in zip(shapes, gold["scales"])]
    cfg = dict(CFG, lr=gold["lr_first"], clipping_update_period=gold["clipping_update_period"])
    dflt = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                          # the oracle's own state (sg, sv, norms) in float64 too
    try:
        oo = gpt_oracle.ScaledAdamOracle([t.clone() for t in init], lr=gold["lr_first"],
                                         clipping_update_period=gold["clipping_update_period"])
        _sadam_vs_oracle(gold, shapes, init, cfg, oo)
    finally:
        torch.set_default_dtype(dflt)


def _sadam_vs_oracle(gold, shapes, init, cfg, oo):
    g0 = _gen(gold["seed"])
    for s in shapes:
        torch.randn(s, generator=g0, dtype=torch.float32)            # the draws of the initial parameters
    p = [t.clone() for t in init]
    delta, v = [torch.zeros_like(t) for t in p], [torch.zeros_like(t) for t in p]
    st = fresh_state(len(p), cfg)
    lr, cs_seen = gold["lr_first"], 1.0
    for it in range(gold["steps"]):
        grads = [(torch.randn(s, generator=g0, dtype=torch.float32) * (5.0 if it in gold["big_grad_steps"] else 1.0)).double() for s in shapes]
        out, _ = T.sadam_step(p, grads, delta, v, st, cfg, lr, as_f32=False)
        cs = oo.step(grads)
        cs_seen = min(cs_seen, float(cs))
        assert abs(float(out["cs"].v) - float(cs)) <= 1e-12
        p = [x.v.reshape(s) for x, s in zip(out["p"], shapes)]
        delta = [x.v.reshape(s) for x, s in zip(out["delta"], shapes)]
        v = [x.v.reshape(s) for x, s in zip(out["v"], shapes)]
        st = dict(step=out["step"], rms=out["rms"].v, sv=out["sv"].v, sg=out["sg"].v, norms=out["norms"].v, thr=out["thr"].v)
        for a, b in zip(p, oo.params):
            assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max())), f"step {it}"
        if it == 0:
            lr = oo.lr = gold["lr_rest"]
    assert cs_seen < 1.0                                              # the schedule reaches the clipping branch


def sadam_case(case):
    """inputs of one injected-state ScaledAdam step: (p, g, delta, v, state, cfg, lr, gscale); shared with the GPU test"""
    g0 = _gen(case["seed"])
    cfg = dict(CFG, **case.get("cfg", {}))
    shapes = case["shapes"]
    nt, sup, per = len(shapes), cfg["size_update_period"], cfg["clipping_update_period"]
    p = [torch.randn(s, generator=g0) * sc for s, sc in zip(shapes, case["scales"])]
    g = [torch.randn(s, generator=g0) * case.get("gmul", 1.0) for s in shapes]
    delta = [torch.randn(s, generator=g0) * 1e-3 for s in shapes]
    v = [torch.rand(s, generator=g0) * 1e-2 for s in shapes]
    st = dict(step=case["step"], rms=torch.rand(nt, generator=g0) + 0.5, sv=torch.rand(nt, generator=g0) * 1e-2,
              sg=torch.randn(sup, nt, generator=g0), norms=torch.rand(per, generator=g0) * 20 + 5,
              thr=torch.tensor([case.get("thr", 0.0), 1.0 if case.get("thr") is not None else 0.0]))
    return p, g, delta, v, st, cfg, case.get("lr", 0.002), case.get("gscale", 1.0)


def test_sadam_emulation_within_model_and_faults():
    case = dict(seed=5, step=15, shapes=[(6, 5), (3 * 8192 + 5,), (1,), (40,)], scales=[1.0, 0.05, 4.0, 5.0],
                cfg=dict(clipping_update_period=8), thr=3.0, gscale=0.5)
    p, g, delta, v, st, cfg, lr, gs = sadam_case(case)
    out, dec = T.sadam_step(p, g, delta, v, st, cfg, lr, gs)
    for what, margin, bound in dec:
        assert margin > R.SAFETY * bound, what
    em = T.emulate_sadam(p, g, delta, v, st, cfg, lr, gs)
    for t in range(len(p)):
        within_model(em["p"][t], out["p"][t], "p")
        within_model(em["delta"][t], out["delta"][t], "delta")
        within_model(em["v"][t], out["v"][t], "v")
    for k in ("rms", "sv", "sg", "coef", "norms"):
        within_model(em[k], out[k], k)
    # a clipping-update step at period 7: the median index min(6, 2) = 2 against 3
    case = dict(seed=6, step=14, shapes=[(6, 5), (40,)], scales=[1.0, 1.0], cfg=dict(clipping_update_period=7), gmul=30.0)
    p, g, delta, v, st, cfg, lr, gs = sadam_case(case)
    out, _ = T.sadam_step(p, g, delta, v, st, cfg, lr, gs)
    em = T.emulate_sadam(p, g, delta, v, st, cfg, lr, gs, median_idx=lambda per: (per // 4) * 2 + 1)
    outside(em["thr"][:1], out["thr"][:1], "clipping median one slot up")
    # a size-update step with rms > param_max_rms
    case = dict(seed=7, step=7, shapes=[(6, 5)], scales=[5.0])
    p, g, delta, v, st, cfg, lr, gs = sadam_case(case)
    out, _ = T.sadam_step(p, g, delta, v, st, cfg, lr, gs)
    em = T.emulate_sadam(p, g, delta, v, st, cfg, lr, gs, drop_rmax=True)
    outside(em["p"][0], out["p"][0], "param_max_rms override dropped")


# ---- nearest code and quantizer ------------------------------------------------------------------------------------------------
def test_sgemm_and_distance_emulation_within_model():
    g0 = _gen(11)
    x, e = torch.randn(37, 70, generator=g0), torch.randn(45, 70, generator=g0)
    within_model(T.emulate_sgemm_nt(x, e), T.sgemm_nt(x, e), "sgemm")
    within_model(T.emulate_vq_dist(x, e), T.vq_dist(x, e), "distance")


def test_nearest_reference_matches_oracle():
    g0 = _gen(12)
    x, e = torch.randn(300, 64, generator=g0), torch.randn(100, 64, generator=g0)
    codes = T.first_argmax(T.vq_dist(x, e).v)
    assert torch.equal(codes, vq_train_oracle.nearest(x.double(), e.double()))


def test_integer_ties_pick_the_lowest_index():
    x = torch.tensor([[1.0, 0.0], [0.0, 0.0], [2.0, 2.0]])
    e = torch.tensor([[0.0, 1.0], [1.0, 0.0], [1.0, 0.0], [-1.0, 0.0], [0.0, -1.0]])
    d = T.vq_dist(x, e)
    assert float(d.e.max()) > 0 and torch.equal(T.first_argmax(d.v), torch.tensor([1, 0, 0]))


def ema_inputs(seed, B=3, T2=11, D=20, K=9, rows_ref=8):
    g0 = _gen(seed)
    x = torch.randn(B, T2, D, generator=g0)
    codes = torch.randint(0, K - 1, (B, T2), generator=g0)           # code K - 1 is never picked
    cs, ea = torch.rand(K, generator=g0) * 3, torch.randn(K, D, generator=g0)
    return x, codes, rows_ref, cs, ea


def test_vq_ema_emulation_within_model_and_fault():
    x, codes, rr, cs, ea = ema_inputs(13)
    ref = T.vq_ema(x, codes, rr, cs, ea, 0.99, 1e-5)
    em = T.emulate_vq_ema(x, codes, rr, cs, ea, 0.99, 1e-5)
    for a, b, w in zip(em, ref, ("cluster_size", "embed_avg", "embed")):
        within_model(a, b, w)
    bad = T.emulate_vq_ema(x, codes, rr, cs, ea, 0.99, 1e-5, count_all_rows=True)
    outside(bad[0], ref[0], "EMA counts rows past rows_ref")


def test_vq_ema_reference_matches_oracle():
    x, codes, _, cs, ea = ema_inputs(14, rows_ref=11)
    ref = T.vq_ema(x, codes, 11, cs, ea, vq_train_oracle.DECAY, vq_train_oracle.EPS)
    D, K = x.shape[-1], cs.shape[0]
    o = vq_train_oracle.ema(dict(cluster_size=cs, embed_avg=ea, embed=torch.zeros(K, D), inited=torch.ones(1)),
                            x.reshape(-1, D), codes.reshape(-1))                 # the oracle is fp32 torch
    for k, r in (("cluster_size", ref[0]), ("embed_avg", ref[1]), ("embed", ref[2])):
        assert float((r.v - o[k].double()).abs().max()) <= 1e-5 * max(1.0, float(o[k].abs().max())), k


def test_straight_through_reference_matches_oracle_step():
    """oracle step's commit loss (kl_ssl) and codes on an inited codebook against vq_commit_loss / vq_dist"""
    cfg = dict(seed=15, B=2, D=16, T=14, steps=1)
    w, b, ssls, ups = vq_train_oracle.pin_inputs(cfg)
    K, rr = 12, 5
    embed = torch.randn(K, cfg["D"], generator=_gen(16)) * 0.3
    buf = dict(embed=embed, embed_avg=embed.clone(), cluster_size=torch.ones(K), inited=torch.ones(1))
    o = vq_train_oracle.step(ssls[0], w, b, buf, ups[0], rows_ref=rr)
    xc = torch.nn.functional.conv1d(ssls[0][:, :, :2 * rr], w, b, stride=2).transpose(1, 2)      # [B, rr, D]
    codes = T.first_argmax(T.vq_dist(xc.reshape(-1, cfg["D"]), embed).v)
    assert torch.equal(codes.reshape(cfg["B"], rr), o["codes"])
    x = torch.zeros(cfg["B"], 7, cfg["D"])
    x[:, :rr] = xc
    q = embed[0].expand(cfg["B"], 7, cfg["D"]).clone()
    q[:, :rr] = embed[codes].reshape(cfg["B"], rr, -1)
    qst = T.vq_st_fwd_emulate(x, q)
    kl = T.vq_commit_loss(x, qst, rr)
    assert abs(float(kl.v) - float(o["kl_ssl"])) <= R.SAFETY * float(kl.e) + 1e-6 * float(o["kl_ssl"])


@pytest.mark.parametrize("rows", [1, 63, 64, 65, 1000, 4097])
def test_col_sum_emulation_within_model(rows):
    x = torch.randn(rows, 37, generator=_gen(rows))
    within_model(T.emulate_col_sum(x), T.col_sum(x), "col_sum")
