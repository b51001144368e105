"""Every output of the weight-norm packing (csrc/pack.cu), ScaledAdam (csrc/gpt_misc.cu) and nearest-code / trainable
quantizer kernels (csrc/vq_loss_optim.cu, csrc/vq_train.cu) against float64, element for element, with the per-element
bounds of tests/train_ref.py (gate = SAFETY x model; a TF32-rounded value adds half a TF32 ulp).

The conventions are tests/test_gpu_cudacore_elementwise.py's, whose buffer helpers this file uses: operands sit in
pitch-padded buffers with NaN in the padding, outputs are pre-filled with NaN and their padding with SENTINEL, and every
case runs twice from the same inputs and must give the same bits.  Branch decisions (the ScaledAdam size-update overrides,
the clipping median and scale, the nearest code) are asserted to sit farther from their threshold than the bound, or are
checked by the rule that holds when they do not.
"""
import ctypes

import pytest
import torch

from tests import cudacore_ref as R
from tests import train_ref as T
from tests.test_cpu_train_ref import sadam_case
from tests.test_gpu_cudacore_elementwise import NAN, SENTINEL, P, bits, body, operand, output, twice

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
WORST = {}


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init()
    try:
        yield ops
    finally:
        for k in sorted(WORST):
            print(f"worst err / gate  {k}: {WORST[k]:.3f}")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def check(got, ref, what, extra=None):
    """|got - ref.v| <= SAFETY ref.e (+ extra) at every element (bit-exact where both are 0); records err / gate"""
    got = got.double().reshape(ref.v.shape)
    gate = R.SAFETY * ref.e + (0.0 if extra is None else extra)
    err = (got - ref.v).abs()
    bad = ~torch.isfinite(got) | (err > gate)
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[:6].tolist()
        lines = [f"  {tuple(i)}: got {float(got[tuple(i)])!r} want {float(ref.v[tuple(i)])!r} gate {float(gate[tuple(i)]):.3g}"
                 for i in idx]
        pytest.fail(f"{what}: {n} of {bad.numel()} outside the gate\n" + "\n".join(lines))
    w = float(torch.where(err == 0, torch.zeros_like(err), err / gate.clamp_min(1e-300)).max()) if got.numel() else 0.0
    k = what.split(" ")[0]
    WORST[k] = max(WORST.get(k, 0.0), w)


def guarded(x, guard=64):
    """a contiguous device copy of x inside a NaN-filled buffer (NaN before and after): a read past x poisons an output"""
    buf = torch.full((x.numel() + 2 * guard,), NAN)
    buf[guard:guard + x.numel()] = x.reshape(-1)
    buf = buf.to(DEV)
    return buf, buf[guard:guard + x.numel()].view(x.shape)


def set_precise(on):
    from easevoice_trainer_b200 import lib
    L = lib.init()
    old = L.evk_get_precise()
    L.evk_set_precise(int(on))
    return old


# ---- weight-norm packing ------------------------------------------------------------------------------------------------------
# (D0, D1, Q, pad0, pad1): Linear, k = 3 / 5 / 7 convs, a ConvTranspose weight [Cin, Cout, k], D0 < 4 padded to 4, D1 < 4
# padded to 4 (both pitch-padded to a multiple of 4), a 6-element row (< 256) and a 1500-element row (> 256 * 5)
PACK_CASES = [(48, 40, 1, 0, 0), (32, 16, 3, 0, 0), (24, 13, 5, 0, 0), (8, 20, 7, 0, 0), (16, 6, 4, 0, 0), (2, 16, 3, 4, 0),
              (16, 1, 7, 0, 4), (3, 2, 3, 4, 4), (4, 300, 5, 0, 0)]
PACK_IDS = ["linear", "k3", "k5", "k7", "convT", "D0_2-pad0", "D1_1-pad1", "D0_3-D1_2-pads", "row1500"]


def pack_inputs(D0, D1, Q, seed):
    g0 = _gen(seed)
    v = torch.randn(D0, D1, Q, generator=g0)
    v[0] *= 1e-3                                                      # a small-norm row
    g = torch.rand(D0, generator=g0) + 0.5
    dpa = torch.randn(Q, D0, D1, generator=g0)
    return v, g, dpa


def pack_job(ops, v, g, D0, D1, Q, D0p, D1p, lda, ldb, pa, pb, dpa=None, dv=None, dg=None):
    from easevoice_trainer_b200 import lib
    return lib.PackJob(v=v.data_ptr(), g=g.data_ptr() if g is not None else None, pa=pa.data_ptr() if pa is not None else None,
                       pb=pb.data_ptr() if pb is not None else None, dpa=dpa.data_ptr() if dpa is not None else None,
                       dv=dv.data_ptr() if dv is not None else None, dg=dg.data_ptr() if dg is not None else None,
                       D0=D0, D1=D1, Q=Q, lda=lda, D0p=D0p, ldb=ldb, D1p=D1p, row0=0)


def packed_out(Q, Dp, ld, D, Dx):
    """[Q, Dp, ld] with NaN where the kernel must write (rows < Dx, columns < D) and SENTINEL in the padding"""
    b = torch.full((Q, Dp, ld), SENTINEL)
    b[:, :Dx, :D] = NAN
    return b.to(DEV)


def pa_rows(pa, D0, D1, Q):
    """pa [Q, D0p, lda] -> [D0, D1 Q] in v's order"""
    return pa[:, :D0, :D1].permute(1, 2, 0).reshape(D0, D1 * Q)


@pytest.mark.parametrize("precise", [False, True], ids=["tf32", "precise"])
@pytest.mark.parametrize("case", PACK_CASES, ids=PACK_IDS)
def test_weight_pack(ops, case, precise):
    D0, D1, Q, pad0, pad1 = case
    v, g, dpa = pack_inputs(D0, D1, Q, D0 * 100 + D1 * 10 + Q)
    _, _, _, D0p, D1p, lda, ldb = ops._pack_geometry(v, pad0, pad1)
    n = D1 * Q
    old = set_precise(precise)
    try:
        for with_g in (True, False):
            gg = g if with_g else None

            def run():
                _vb, vd = guarded(v)
                _gb, gd = guarded(g)
                pa, pb = packed_out(Q, D0p, lda, D1, D0), packed_out(Q, D1p, ldb, D0, D1)
                job = pack_job(ops, vd, gd if with_g else None, D0, D1, Q, D0p, D1p, lda, ldb, pa, pb)
                P(_vb); P(_gb)
                ops._call("evk_weight_pack_one", ctypes.byref(job))
                return [pa.cpu(), pb.cpu()]

            pa, pb = twice(run)
            pad_a, pad_b = torch.ones_like(pa, dtype=torch.bool), torch.ones_like(pb, dtype=torch.bool)
            pad_a[:, :D0, :D1] = False
            pad_b[:, :D1, :D0] = False
            assert bool((pa[pad_a] == SENTINEL).all()) and bool((pb[pad_b] == SENTINEL).all()), "padding was written"
            got = pa_rows(pa, D0, D1, Q)
            assert torch.equal(bits([pb[:, :D1, :D0].permute(2, 1, 0).reshape(D0, n)])[0], bits([got])[0]), "pb != pa^T"
            ref = T.weight_pack(v.reshape(D0, n), gg)
            tag = f"weight_pack_{'precise' if precise else 'tf32'} D0={D0} D1={D1} Q={Q} g={with_g}"
            if precise:
                check(got, ref, tag)
            else:
                assert bool(((got.contiguous().view(torch.int32) & 0x1FFF) == 0).all()), f"{tag}: a value is not TF32"
                check(got, ref, tag, T.tf32_gate(ref, R.SAFETY))
            # the library's wrapper: the same bits, and its zero-allocated channel and pitch padding stays exactly zero
            pw = ops.pack_weight(v.to(DEV), g.to(DEV) if with_g else None, True, pad0, pad1)
            wa, wb = pw.pa.cpu(), pw.pb.cpu()
            assert torch.equal(bits([wa[~pad_a]])[0], bits([pa[~pad_a]])[0]) and bool((wa[pad_a] == 0).all())
            assert torch.equal(bits([wb[~pad_b]])[0], bits([pb[~pad_b]])[0]) and bool((wb[pad_b] == 0).all())
    finally:
        set_precise(old)


@pytest.mark.parametrize("case", PACK_CASES, ids=PACK_IDS)
def test_weight_pack_bwd(ops, case):
    D0, D1, Q, pad0, pad1 = case
    v, g, dpa = pack_inputs(D0, D1, Q, D0 * 100 + D1 * 10 + Q + 1)
    _, _, _, D0p, D1p, lda, ldb = ops._pack_geometry(v, pad0, pad1)
    n = D1 * Q
    dpa_buf = torch.full((Q, D0p, lda), NAN)
    dpa_buf[:, :D0, :D1] = dpa
    for with_g in (True, False):
        def run():
            _vb, vd = guarded(v)
            _gb, gd = guarded(g)
            dd = dpa_buf.to(DEV)
            dvb, dv = guarded(torch.full((D0, D1, Q), NAN))
            dgb, dg = guarded(torch.full((D0,), NAN))
            dvb[:64] = SENTINEL; dvb[-64:] = SENTINEL; dgb[:64] = SENTINEL; dgb[-64:] = SENTINEL
            job = pack_job(ops, vd, gd if with_g else None, D0, D1, Q, D0p, D1p, lda, ldb, None, None, dd, dv, dg if with_g else None)
            P(_vb); P(_gb); P(dd); P(dvb); P(dgb)
            ops._call("evk_weight_pack_bwd_one", ctypes.byref(job))
            return [dvb.cpu(), dgb.cpu()]

        dvb, dgb = twice(run)
        assert bool((dvb[:64] == SENTINEL).all()) and bool((dvb[-64:] == SENTINEL).all()), "dv written outside its rows"
        dv, dg = dvb[64:-64].reshape(D0, n), dgb[64:-64]
        dpa_rows = dpa.permute(1, 2, 0).reshape(D0, n)
        if not with_g:
            assert torch.equal(bits([dv])[0], bits([dpa_rows.contiguous()])[0]), "g = None: dv must be dpa bit for bit"
            assert bool(torch.isnan(dg).all()), "g = None: dg was written"
            continue
        rdv, rdg = T.weight_pack_bwd(v.reshape(D0, n), g, dpa_rows)
        check(dv, rdv, f"weight_pack_bwd dv D0={D0} D1={D1} Q={Q}")
        check(dg, rdg, f"weight_pack_bwd dg D0={D0} D1={D1} Q={Q}")


# (D0, D1, Q, with g, need_pb, pad0, pad1, wants_grad).  Frozen jobs sit between wanted ones, so the backward table's row0
# must count only wanted rows.  The 1500-element row comes first and every later job's rows are short, so a job table
# whose row0 were not re-based would still address inside the arenas (and be caught by the bit comparisons below).
PLAN = [(4, 300, 5, True, False, 0, 0, True), (16, 12, 3, True, True, 0, 0, True), (24, 40, 5, True, False, 0, 0, False),
        (8, 20, 1, True, True, 0, 0, True), (2, 16, 3, False, True, 4, 0, True), (16, 1, 7, True, True, 0, 4, False),
        (12, 8, 4, True, True, 0, 0, True), (10, 6, 3, False, False, 0, 0, False), (6, 10, 7, True, True, 0, 0, True)]


def plan_params(spec, seed):
    """every v and g as a view of one flat parameter arena (as the trainers' optimizers hold them), NaN between them"""
    g0 = _gen(seed)
    sizes = [(D0 * D1 * Q, D0 if wg else 0) for D0, D1, Q, wg, *_ in spec]
    arena = torch.full((4096 + sum(a + b + 64 for a, b in sizes),), NAN, device=DEV)
    off, vs, gs = 4096, [], []
    for (D0, D1, Q, wg, *_), (nv, ng) in zip(spec, sizes):
        v = arena[off:off + nv].view(D0, D1, Q)
        v.copy_(torch.randn(D0, D1, Q, generator=g0))
        off += nv + 32
        g = None
        if wg:
            g = arena[off:off + ng]
            g.copy_(torch.rand(D0, generator=g0) + 0.5)
            off += ng + 32
        vs.append(v); gs.append(g)
    return arena, vs, gs


@pytest.mark.parametrize("frozen_all", [False, True], ids=["mixed", "no_grad_wanted"])
def test_pack_plan_table(ops, frozen_all):
    spec = [s[:7] + (False if frozen_all else s[7],) for s in PLAN]
    arena, vs, gs = plan_params(spec, 21)
    reqs = [(f"w{i}", v, g, s[4], s[5], s[6], s[7]) for i, (s, v, g) in enumerate(zip(spec, vs, gs))]
    plan = ops.PackPlan(reqs, with_grad=True)
    g0 = _gen(22)
    dpas = []
    for dp in plan.dpa:                                                # the packed gradients, NaN in their padding
        Q, D0p, lda = dp.shape
        dpas.append(torch.randn(Q, D0p, lda, generator=g0))

    def run():
        plan.arena_pa.fill_(NAN)
        plan.arena_pb.fill_(NAN)
        packed = ops.pack_all(plan)
        out = [t for pw in packed for t in (pw.pa.detach().cpu(), pw.pb.cpu() if pw.pb is not None else torch.zeros(0))]
        for i, (dp, s) in enumerate(zip(plan.dpa, spec)):
            x = torch.full(dp.shape, NAN)
            x[:, :s[0], :s[1]] = dpas[i][:, :s[0], :s[1]]
            dp.copy_(x.to(DEV))
        plan.arena_dvg.fill_(SENTINEL)
        plan.run_pack_bwd()
        return out + [plan.arena_dvg.cpu()]

    res = twice(run)
    dvg = res[-1]
    written = torch.zeros_like(dvg, dtype=torch.bool)
    base = plan.arena_dvg.data_ptr()
    for i, (s, v, g) in enumerate(zip(spec, vs, gs)):
        D0, D1, Q, wg, need_pb, pad0, pad1, wants = s
        pw = ops.pack_weight(v, g, need_pb, pad0, pad1)
        pa, pb = res[2 * i], res[2 * i + 1]
        sel = torch.zeros_like(pa, dtype=torch.bool)
        sel[:, :D0, :D1] = True
        assert torch.equal(bits([pa[sel]])[0], bits([pw.pa.detach().cpu()[sel]])[0]), f"job {i}: pack_all pa != pack_weight"
        if need_pb:
            selb = torch.zeros_like(pb, dtype=torch.bool)
            selb[:, :D1, :D0] = True
            assert torch.equal(bits([pb[selb]])[0], bits([pw.pb.cpu()[selb]])[0]), f"job {i}: pack_all pb != pack_weight"
    # each job's dv / dg slice of the arena, read back from the plan's job table
    from easevoice_trainer_b200 import lib
    jobs = (lib.PackJob * len(spec)).from_buffer_copy(bytes(plan.jobs.cpu().numpy().tobytes()))
    for i, (s, v, g) in enumerate(zip(spec, vs, gs)):
        D0, D1, Q, wg, need_pb, pad0, pad1, wants = s
        o_dv = (jobs[i].dv - base) // 4
        o_dg = (jobs[i].dg - base) // 4 if wg else None
        dv_got = dvg[o_dv:o_dv + D0 * D1 * Q]
        if not wants:
            assert bool((dv_got == SENTINEL).all()), f"frozen job {i}: its dv slice was written"
            if wg:
                assert bool((dvg[o_dg:o_dg + D0] == SENTINEL).all()), f"frozen job {i}: its dg slice was written"
            continue
        written[o_dv:o_dv + D0 * D1 * Q] = True
        vr = v.clone().requires_grad_(True)
        gr = g.clone().requires_grad_(True) if wg else None
        pw = ops.pack_weight(vr, gr, need_pb, pad0, pad1)
        x = torch.full(pw.pa.shape, NAN)
        x[:, :D0, :D1] = dpas[i][:, :D0, :D1]
        grads = torch.autograd.grad(pw.pa, [vr] + ([gr] if wg else []), x.to(DEV))      # evk_weight_pack_bwd_one
        assert torch.equal(bits([dv_got])[0], bits([grads[0].cpu().reshape(-1)])[0]), f"job {i}: table dv != _bwd_one"
        if wg:
            written[o_dg:o_dg + D0] = True
            assert torch.equal(bits([dvg[o_dg:o_dg + D0]])[0], bits([grads[1].cpu()])[0]), f"job {i}: table dg != _bwd_one"
    assert bool((dvg[~written] == SENTINEL).all()), "the backward table wrote outside the wanted jobs' dv / dg slices"
    if frozen_all:
        assert plan.rows_bwd.numel() == 0
    del arena


# ---- ScaledAdam -------------------------------------------------------------------------------------------------------------------
BIG = 3 * 8192 + 5                 # four chunks of the chunk table, the last one 5 elements
SADAM_CASES = {
    # step 0: the rms init, no clipping; a 4-chunk tensor and a scalar
    "step0": dict(seed=1, step=0, shapes=[(6, 5), (BIG,), (1,)], scales=[1.0, 0.05, 2.0]),
    # a size-update step (step % 4 == 3) with one tensor below param_min_rms, one above param_max_rms and one between
    "size_update": dict(seed=2, step=7, shapes=[(6, 5), (40,), (BIG,)], scales=[1e-6, 5.0, 1.0]),
    # clipping-update steps: the median index min(period - 1, (period / 4) * 2) is 0, 0, 2 and 500
    "clip_period1": dict(seed=3, step=5, shapes=[(6, 5), (40,)], scales=[1.0, 1.0], cfg=dict(clipping_update_period=1)),
    "clip_period3": dict(seed=4, step=6, shapes=[(6, 5), (40,)], scales=[1.0, 1.0], cfg=dict(clipping_update_period=3)),
    "clip_period7": dict(seed=5, step=14, shapes=[(6, 5), (40,)], scales=[1.0, 1.0], cfg=dict(clipping_update_period=7)),
    "clip_period1000": dict(seed=6, step=2000, shapes=[(6, 5), (BIG,), (1,)], scales=[1.0, 0.05, 1.0], gmul=3.0),
    # clipping engaged: threshold 2 against a gradient norm near 10
    "clip_engaged": dict(seed=7, step=13, shapes=[(6, 5), (40,)], scales=[1.0, 1.0], cfg=dict(clipping_update_period=8), thr=2.0),
    # bc2 = 1 - 0.95^(step + 1) crosses 0.99 between steps 88 and 89
    "bc2_below": dict(seed=8, step=88, shapes=[(6, 5), (1,)], scales=[1.0, 1.0]),
    "bc2_above": dict(seed=9, step=89, shapes=[(6, 5), (1,)], scales=[1.0, 1.0]),
    # scalar parameters beyond +-scalar_max, a size update and gscale != 1
    "scalars_gscale": dict(seed=10, step=11, shapes=[(1,), (1,), (BIG,), (7,)], scales=[14.0, 14.0, 0.05, 1.0], gscale=0.25),
}
SADAM_RUNS = [(k, zg) for k in SADAM_CASES for zg in (True, False)]


@pytest.mark.parametrize("name,zero_grad", SADAM_RUNS, ids=[f"{k}-zero_grad{int(z)}" for k, z in SADAM_RUNS])
def test_scaled_adam_step(ops, name, zero_grad):
    from easevoice_trainer_b200.train.gpt_step import FlatScaledAdam
    case = SADAM_CASES[name]
    p, g, delta, v, st, cfg, lr, gscale = sadam_case(case)
    if name == "scalars_gscale":
        p[0].fill_(12.5); p[1].fill_(-15.0)
    ref, dec = T.sadam_step(p, g, delta, v, st, cfg, lr, gscale)
    for what, margin, bound in dec:                       # every branch the step takes is decided beyond its bound
        assert margin > R.SAFETY * bound, f"{name}: {what}: margin {margin:.3g} <= gate {R.SAFETY * bound:.3g}"
    kw = {k: v_ for k, v_ in cfg.items() if k != "lr"}
    opt = FlatScaledAdam([(f"p{i}", torch.nn.Parameter(t.clone().to(DEV))) for i, t in enumerate(p)], lr=lr, **kw)
    cat = lambda ts: torch.cat([t.reshape(-1) for t in ts]).to(DEV)

    def run():
        opt.flat_p.copy_(cat(p)); opt.flat_g.copy_(cat(g)); opt.flat_delta.copy_(cat(delta)); opt.flat_v.copy_(cat(v))
        opt.rms.copy_(st["rms"]); opt.sv.copy_(st["sv"]); opt.sg.copy_(st["sg"]); opt.norms.copy_(st["norms"])
        opt.thr.copy_(st["thr"]); opt.stepbuf.fill_(st["step"]); opt.set_lr(lr)
        opt.glob.fill_(NAN); opt.coef.fill_(NAN)
        opt.step(gscale, zero_grad)
        return [opt.flat_p.cpu(), opt.flat_g.cpu(), opt.flat_delta.cpu(), opt.flat_v.cpu(), opt.rms.cpu(), opt.sv.cpu(),
                opt.sg.cpu(), opt.coef.cpu(), opt.glob.cpu(), opt.norms.cpu(), opt.thr.cpu(), opt.stats.cpu(), opt.stepbuf.cpu()]

    fp, fg, fd, fv, rms, sv, sg, coef, glob, norms, thr, stats, stepbuf = twice(run)
    off = 0
    for t, tp in enumerate(p):
        k = tp.numel()
        check(fp[off:off + k], ref["p"][t], f"sadam_update p {name} tensor {t}")
        check(fd[off:off + k], ref["delta"][t], f"sadam_update delta {name} tensor {t}")
        check(fv[off:off + k], ref["v"][t], f"sadam_update v {name} tensor {t}")
        off += k
    if zero_grad:
        assert bool((fg == 0).all())
    else:
        assert torch.equal(bits([fg])[0], bits([cat(g).cpu()])[0])
    for what, got in (("rms", rms), ("sv", sv), ("sg", sg), ("coef", coef), ("norms", norms), ("thr", thr)):
        check(got, ref[what], f"sadam_scalars {what} {name}")
    check(glob[:3], ref["glob"], f"sadam_scalars glob {name}")
    assert bool((stats == 0).all()) and int(stepbuf[0]) == st["step"] + 1


# ---- nearest code ---------------------------------------------------------------------------------------------------------------
SGEMM_CASES = [(1, 1, 1), (65, 63, 1), (70, 130, 5), (129, 67, 17), (33, 1024, 768)]


@pytest.mark.parametrize("M,N,K", SGEMM_CASES, ids=[f"M{m}-N{n}-K{k}" for m, n, k in SGEMM_CASES])
def test_sgemm_nt_f32(ops, M, N, K):
    g0 = _gen(M * 7 + N + K)
    a, b = torch.randn(M, K, generator=g0), torch.randn(N, K, generator=g0)

    def run():
        ad, bd = operand(a, K + 3), operand(b, K + 1)
        c = output(M, N, N + 2)
        ops._call("evk_sgemm_nt_f32", P(ad), K + 3, P(bd), K + 1, P(c), N + 2, M, N, K)
        return [body(c, N, "sgemm_nt C")]

    (c,) = twice(run)
    check(c, T.sgemm_nt(a, b), f"sgemm_nt_f32 M={M} N={N} K={K}")


def nearest_direct(ops, x, e):
    """sgemm_nt_f32 + vq_argmax with pitch-padded operands -> codes"""
    rows, D = x.shape
    K = e.shape[0]
    xd, ed = operand(x, D + 1), operand(e, D + 3)
    dots = output(rows, K, K + 2)
    ops._call("evk_sgemm_nt_f32", P(xd), D + 1, P(ed), D + 3, P(dots), K + 2, rows, K, D)
    codes = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
    scratch = torch.full((K,), NAN, device=DEV)
    ops._call("evk_vq_argmax", P(dots), K + 2, P(xd), D + 1, P(ed), D + 3, rows, K, D, P(codes), P(scratch))
    return [codes.cpu()]


def nearest_inputs(kind, seed):
    g0 = _gen(seed)
    if kind == "codebook":                                            # the real 1024 x 768 codebook shape
        e = torch.randn(1024, 768, generator=g0)
        x = torch.randn(300, 768, generator=g0)
    else:                                                             # near-ties: midpoints of codeword pairs, ~1e-6 apart
        e = torch.randn(300, 64, generator=g0)
        i, j = torch.randint(0, 300, (200,), generator=g0), torch.randint(0, 300, (200,), generator=g0)
        x = 0.5 * (e[i] + e[j]) + 1e-6 * torch.randn(200, 64, generator=g0)
    return x, e


@pytest.mark.parametrize("kind", ["codebook", "near_ties"])
def test_vq_nearest(ops, kind):
    x, e = nearest_inputs(kind, 31)
    (codes,) = twice(lambda: nearest_direct(ops, x, e))
    assert torch.equal(codes, ops.vq_nearest(x.to(DEV)[None], e.to(DEV))[0].cpu())
    d = T.vq_dist(x, e)
    best = T.first_argmax(d.v)
    r = torch.arange(x.shape[0])
    # the chosen code's fp32 distance beat the float64 best's: d64[best] - d64[code] <= gate(code) + gate(best)
    lost = d.v[r, best] - d.v[r, codes]
    allow = R.SAFETY * (d.e[r, codes] + d.e[r, best])
    assert bool((lost <= allow).all()), f"{int((lost > allow).sum())} rows picked a code beyond the bound of the minimum"
    # where the gap to the runner-up exceeds both bounds the code is the float64 argmin
    d2 = d.v.clone()
    d2[r, best] = -float("inf")
    second = d2.argmax(-1)
    decided = (d.v[r, best] - d.v[r, second]) > R.SAFETY * (d.e[r, best] + d.e[r, second])
    assert torch.equal(codes[decided], best[decided])
    print(f"vq_nearest {kind}: {int(decided.sum())} of {len(r)} rows decided beyond the bound")
    # random rows on the real codebook are decided; the midpoints exercise the rule for rows that are not
    assert int(decided.sum()) > 0 if kind == "codebook" else int(decided.sum()) < len(r)
    WORST["vq_argmax"] = max(WORST.get("vq_argmax", 0.0), float((lost / allow.clamp_min(1e-300)).clamp_min(0).max()))


def test_vq_argmax_exact_ties_pick_lowest_index(ops):
    """integer operands make every distance exact: ties and duplicate codewords (spread over threads and warps: code k and
    k + 300 are equal) must return the lowest index, like torch.max"""
    g0 = _gen(41)
    e = torch.randint(-2, 3, (600, 6), generator=g0).float()
    e[300:] = e[:300]
    x = torch.randint(-2, 3, (257, 6), generator=g0).float()
    (codes,) = twice(lambda: nearest_direct(ops, x, e))
    d = T.vq_dist(x, e).v
    want = T.first_argmax(d)
    ties = ((d == d.max(-1, keepdim=True).values).sum(-1) > 1).sum()
    assert int(ties) == x.shape[0]                                   # every row has a tie (at least its duplicate)
    assert torch.equal(codes, want)


# ---- trainable quantizer ---------------------------------------------------------------------------------------------------------
EMA_CASES = [(4, 50, 768, 1024, 37), (3, 11, 300, 9, 8), (2, 7, 20, 5, 7)]


@pytest.mark.parametrize("B,T2,D,K,rows_ref", EMA_CASES, ids=[f"B{b}-T{t}-D{d}-K{k}-ref{r}" for b, t, d, k, r in EMA_CASES])
def test_vq_ema(ops, B, T2, D, K, rows_ref):
    g0 = _gen(B * T2 + D)
    x = torch.randn(B, T2, D, generator=g0)
    x[:, rows_ref:] = NAN                                             # rows past rows_ref must not be read
    codes = torch.randint(0, K - 1, (B, T2), generator=g0)           # code K - 1 is picked by no row
    codes[:, rows_ref:] = 0
    cs, ea = torch.rand(K, generator=g0) * 3, torch.randn(K, D, generator=g0)

    def run():
        xd = operand(x.reshape(-1, D), D + 2)
        csd, ead = cs.to(DEV), ea.to(DEV)
        emb = torch.full((K, D), NAN, device=DEV)
        rr = torch.tensor([rows_ref], dtype=torch.int32, device=DEV)
        ops._call("evk_vq_ema", P(xd), D + 2, P(codes.to(DEV)), B, T2, P(rr), P(csd), P(ead), P(emb), K, D,
                  ctypes.c_float(0.99), ctypes.c_float(1e-5))
        return [csd.cpu(), ead.cpu(), emb.cpu()]

    gcs, gea, gemb = twice(run)
    rcs, rea, remb = T.vq_ema(x, codes, rows_ref, cs, ea, 0.99, 1e-5)
    tag = f"B={B} T2={T2} D={D} K={K}"
    check(gcs, rcs, f"vq_ema cluster_size {tag}")
    check(gea, rea, f"vq_ema embed_avg {tag}")
    check(gemb, remb, f"vq_normalize embed {tag}")


ST_CASES = [(2, 9, 20, 6), (3, 40, 768, 37), (1, 5, 1, 5)]


@pytest.mark.parametrize("B,T2,D,rows_ref", ST_CASES, ids=[f"B{b}-T{t}-D{d}-ref{r}" for b, t, d, r in ST_CASES])
def test_vq_straight_through(ops, B, T2, D, rows_ref):
    g0 = _gen(B + T2 + D)
    x = torch.randn(B, T2, D, generator=g0)
    q = x + 0.1 * torch.randn(B, T2, D, generator=g0)
    q[:, rows_ref:] += 1e3                                            # rows past rows_ref would dominate the loss
    dy = torch.randn(B, 2 * T2, D, generator=g0)
    gloss = 0.75

    def run():
        xd, qd = operand(x.reshape(-1, D), D + 1), operand(q.reshape(-1, D), D + 3)
        rr = torch.tensor([rows_ref], dtype=torch.int32, device=DEV)
        y = torch.full((B, 2 * T2, D), NAN, device=DEV)
        qst = torch.full((B, T2, D), NAN, device=DEV)
        loss = torch.full((1,), NAN, device=DEV)
        ops._call("evk_vq_st_fwd", P(xd), D + 1, P(qd), D + 3, B, T2, D, P(rr), P(y), P(qst), P(loss))
        dx = torch.full((B, T2, D), NAN, device=DEV)
        gl = torch.tensor([gloss], device=DEV)
        ops._call("evk_vq_st_bwd", P(dy.to(DEV)), P(xd), D + 1, P(qst), B, T2, D, P(rr), P(gl), P(dx))
        return [y.cpu(), qst.cpu(), loss.cpu(), dx.cpu()]

    y, qst, loss, dx = twice(run)
    want = T.vq_st_fwd_emulate(x, q)
    assert torch.equal(bits([qst])[0], bits([want])[0]), "qst != x + (q - x) in fp32"
    assert torch.equal(bits([y[:, 0::2].contiguous()])[0], bits([want])[0]) and \
        torch.equal(bits([y[:, 1::2].contiguous()])[0], bits([want])[0]), "an upsampled row != x + (q - x)"
    rl = T.vq_commit_loss(x, want, rows_ref)
    check(loss, R.E(rl.v.reshape(1), rl.e.reshape(1)), f"vq_st_fwd loss B={B} T2={T2} D={D}")
    rdx = T.vq_st_bwd(dy, x, want, rows_ref, gloss)
    assert bool((dx[:, rows_ref:] == 0).all()), "dx past rows_ref must be 0"
    check(dx, rdx, f"vq_st_bwd dx B={B} T2={T2} D={D}")


COLSUM_CASES = [(1, 37), (63, 1), (65, 130), (200, 37), (4097, 768)]


@pytest.mark.parametrize("rows,C", COLSUM_CASES, ids=[f"rows{r}-C{c}" for r, c in COLSUM_CASES])
def test_col_sum(ops, rows, C):
    x = torch.randn(rows, C, generator=_gen(rows + C))

    def run():
        buf, xd = guarded(x)
        out = torch.full((C,), NAN, device=DEV)
        P(buf)
        ops._call("evk_col_sum", P(xd), rows, C, P(out))
        return [out.cpu()]

    (out,) = twice(run)
    check(out, T.col_sum(x), f"col_sum rows={rows} C={C}")
