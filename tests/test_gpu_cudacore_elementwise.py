"""Every output of the fp32 CUDA-core training kernels (LayerNorm, fused-dropout LayerNorm, column sums, activations, gates,
masks, gathers, transposes, embeddings, masked mean, position add, cross-entropy, DPO head, losses, AdamW) against float64,
element for element, with the per-element bound of tests/cudacore_ref.py (gate = SAFETY x model).

Operands sit in pitch-padded buffers whose padding holds NaN, so a read of padding poisons an output.  Outputs that every
element must be written are pre-filled with NaN; their pitch padding holds SENTINEL and must come back untouched; outputs
the kernels accumulate into (ordered_sum adds into dst) start from a random base that the reference adds.  Every case runs
twice from the same inputs and must give the same bits: the fixed-order cross-block sums make the kernels reproducible.
The sizes are chosen to reach each launch path; the arithmetic sits next to each case.
"""
import ctypes

import pytest
import torch

from tests import cudacore_ref as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NAN = float("nan")
SENTINEL = -31337.0
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


_ALIVE = []                      # device operands of the launches in flight: a temporary must outlive its kernel


def P(t):
    if t is None:
        return None
    _ALIVE.append(t)
    return ctypes.c_void_p(t.data_ptr())


# ---- buffers --------------------------------------------------------------------------------------------------------------
def operand(x, ld):
    """[rows, C] cpu -> a device [rows, ld] buffer with NaN in the pitch padding"""
    rows, C = x.shape
    buf = torch.full((rows, ld), NAN)
    buf[:, :C] = x
    return buf.to(DEV)


def output(rows, C, ld, fill=NAN):
    buf = torch.full((rows, ld), SENTINEL)
    buf[:, :C] = fill
    return buf.to(DEV)


def body(buf, C, what):
    """the valid columns of an output buffer; its pitch padding must still hold SENTINEL"""
    b = buf.cpu()
    assert bool((b[:, C:] == SENTINEL).all()), f"{what}: pitch padding was written"
    return b[:, :C]


def bits(ts):
    return [t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t for t in ts]


def twice(run):
    """run() -> list of cpu tensors; a second run from the same inputs must give the same bits"""
    a = run()
    torch.cuda.synchronize()
    _ALIVE.clear()
    b = run()
    torch.cuda.synchronize()
    _ALIVE.clear()
    for i, (u, v) in enumerate(zip(bits(a), bits(b))):
        assert torch.equal(u, v), f"output {i} differs between two identical runs"
    return a


def check(got, ref, what, exact=False):
    """|got - ref| <= SAFETY * model at every element (got == ref bit for bit where the model is 0); records err / gate"""
    got = got.double()
    if exact:
        ref = ref if isinstance(ref, R.E) else R.E(ref.double())
        ref = R.E(ref.v, torch.zeros_like(ref.v))
    bad = R.outside_gate(got, ref)
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[:6].tolist()
        lines = [f"  {tuple(i)}: got {float(got[tuple(i)])!r} want {float(ref.v[tuple(i)])!r} gate {R.SAFETY * float(ref.e[tuple(i)]):.3g}"
                 for i in idx]
        pytest.fail(f"{what}: {n} of {bad.numel()} outside the gate\n" + "\n".join(lines))
    w = float(R.ratio(got, ref).max()) if got.numel() else 0.0
    k = what.split(" ")[0]
    WORST[k] = max(WORST.get(k, 0.0), w)
    return w


def row_E(e, rows):
    return R.E(e.v.expand(rows, -1), e.e.expand(rows, -1))


# ---- LayerNorm ------------------------------------------------------------------------------------------------------------
def ln_inputs(rows, C, seed, dc_row=True):
    g = _gen(seed)
    x = torch.randn(rows, C, generator=g)
    x[0] = 0.625                                                     # a constant row: var = 0, y = beta
    if dc_row and rows > 1:
        x[1] = 1e3 + torch.randn(C, generator=g)                     # a large mean: DC 1e3, sigma 1
    res = torch.randn(rows, C, generator=g)
    gamma, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    dy = torch.randn(rows, C, generator=g)
    return x, res, gamma, beta, dy


def ln_fwd(ops, x, res, gamma, beta, eps, rows, C):
    ldx, ldr, ldy = C + 3, C + 5, C + 2
    xd = operand(x, ldx)
    rd = operand(res, ldr) if res is not None else None
    y = output(rows, C, ldy)
    stats = torch.full((rows, 2), NAN, device=DEV)
    ops._call("evk_layernorm_fwd", P(xd), ldx, P(rd), ldr, P(gamma.to(DEV)), P(beta.to(DEV)), eps, P(y), ldy, P(stats), rows, C)
    return body(y, C, "layernorm_fwd y"), stats.cpu()


# (rows, C): rows <= 8 run the block kernel (one 256-thread block per row), rows >= 9 the warp-per-row kernel.  The backward's
# rows_per_block = max(8, ceil(rows / 528)): 4225 rows is the first rpb = 9 (S = 470 blocks), 20000 rows rpb = 38 (S = 527).
LN_CASES = [(r, C) for C in (1, 31, 33, 192, 512, 768, 1023, 1024) for r in (1, 8, 9, 111)] + [(4225, 192), (4225, 768), (20000, 192)]


@pytest.mark.parametrize("rows,C", LN_CASES, ids=[f"rows{r}-C{c}" for r, c in LN_CASES])
def test_layernorm(ops, rows, C):
    with_res = (rows + C) % 2 == 0 or rows == 4225
    eps = 1e-12 if C in (768, 1024, 1023) else 1e-5                 # BERT's eps at its widths
    x, res, gamma, beta, dy = ln_inputs(rows, C, rows * 7 + C)
    r = res if with_res else None
    dgb_base = torch.randn(2, C, generator=_gen(C))

    def run():
        y, stats = ln_fwd(ops, x, r, gamma, beta, eps, rows, C)
        xd, rd = operand(x, C + 3), operand(res, C + 5) if with_res else None
        dyd = operand(dy, C + 1)
        dx = output(rows, C, C + 4)
        dgb = output(2, C, C + 2, 0.0)
        dgb[:, :C] = dgb_base.to(DEV)
        ops._call("evk_layernorm_bwd", P(xd), C + 3, P(rd), C + 5, P(gamma.to(DEV)), P(stats.to(DEV)), P(dyd), C + 1, P(dx), C + 4,
                  P(dgb[0]), P(dgb[1]), rows, C)
        return [y, stats, body(dx, C, "layernorm_bwd dx"), body(dgb, C, "layernorm_bwd dgamma")]

    y, stats, dx, dgb = twice(run)
    t = R.ln_input(x, r)
    ry, rm, rr = R.layernorm_fwd(t, gamma, beta, eps, R.ln_row_chain(C))
    kern = "layernorm_fwd_block" if rows <= 8 else "layernorm_fwd_warp"
    check(y, ry, f"{kern} y rows={rows} C={C}")
    check(stats[:, 0], rm, f"{kern} mean rows={rows} C={C}")
    check(stats[:, 1], rr, f"{kern} rstd rows={rows} C={C}")
    assert float(y[0].sub(beta).abs().max()) == 0.0 or with_res    # constant row: d = 0 exactly, y = beta
    rdx, rdg, rdb = R.layernorm_bwd(t, gamma, stats[:, 0], stats[:, 1], dy, R.ln_row_chain(C), R.ln_param_chain(rows))
    pc = R.ln_param_chain(rows) * R.U32
    check(dx, rdx, f"layernorm_bwd dx rows={rows} C={C}")
    check(dgb[0], R.E(rdg.v + dgb_base[0].double(), rdg.e + pc * dgb_base[0].double().abs()), f"layernorm_bwd dgamma rows={rows} C={C}")
    check(dgb[1], R.E(rdb.v + dgb_base[1].double(), rdb.e + pc * dgb_base[1].double().abs()), f"layernorm_bwd dbeta rows={rows} C={C}")


@pytest.mark.parametrize("C", [33, 192, 512, 1024])
def test_layernorm_rows_8_and_9_agree(ops, C):
    """The block kernel (rows <= 8) takes a row's sums in the warp kernel's order, so a row's bits do not depend on how many
    rows share the launch: the batched KV-cache decoder promises that a row decodes the same alone or in a batch of 9..64."""
    x, res, gamma, beta, _ = ln_inputs(9, C, C)
    y9, s9 = ln_fwd(ops, x, res, gamma, beta, 1e-5, 9, C)
    for rows in (1, 8):
        y, s = ln_fwd(ops, x[:rows], res[:rows], gamma, beta, 1e-5, rows, C)
        assert torch.equal(bits([y])[0], bits([y9[:rows]])[0]), f"C={C}: rows of a {rows}-row launch differ from a 9-row launch"
        assert torch.equal(bits([s])[0], bits([s9[:rows]])[0])


def test_layernorm_refuses_c_1025(ops):
    from easevoice_trainer_b200 import lib
    L = lib.init()
    x = torch.zeros(2, 1025, device=DEV)
    y = torch.full((2, 1025), SENTINEL, device=DEV)
    g = torch.ones(1025, device=DEV)
    rc = L.evk_layernorm_fwd(P(x), 1025, None, 0, P(g), P(g), 1e-5, P(y), 1025, None, 2, 1025, ops._st())
    assert rc == -4 and "C=1025" in lib.last_error()                 # EVK_ERR_UNSUPPORTED
    rc = L.evk_layernorm_bwd(P(x), 1025, None, 0, P(g), P(x), P(x), 1025, P(y), 1025, P(g), P(g), 2, 1025, ops._st())
    assert rc == -4
    torch.cuda.synchronize()
    assert bool((y == SENTINEL).all())                               # refused before any launch


# ---- LayerNorm(x + dropout(res)) ------------------------------------------------------------------------------------------
# contiguous rows only (the kernels read float4 rows of C floats), so no pitch padding; 4300 rows cross rpb > 8 (rpb = 9).
@pytest.mark.parametrize("C,rows", [(4, 37), (192, 4300), (508, 111), (512, 4300)])
def test_layernorm_dropout(ops, C, rows):
    p = 0.1
    x, res, gamma, beta, dy = ln_inputs(rows, C, C + rows, dc_row=False)
    flat = torch.full((2 * C + 3,), NAN)                             # gamma / beta at odd float offsets of flat storage
    flat[1:C + 1], flat[C + 2:2 * C + 2] = gamma, beta
    base = torch.randn(2, C, generator=_gen(3))

    def run():
        ops.manual_seed(1234, DEV)
        rng = ops.rng_state(DEV)
        fd = flat.to(DEV)
        gd, bd = fd[1:C + 1], fd[C + 2:2 * C + 2]
        xd, rd, dyd = x.to(DEV), res.to(DEV), dy.to(DEV)
        y, stats = torch.full((rows, C), NAN, device=DEV), torch.full((rows, 2), NAN, device=DEV)
        ops._call("evk_layernorm_drop_fwd", P(xd), P(rd), P(gd), P(bd), 1e-5, p, P(rng), 5, P(y), P(stats), rows, C)
        dx, dres = torch.full((rows, C), NAN, device=DEV), torch.full((rows, C), NAN, device=DEV)
        dgb = base.to(DEV)
        ops._call("evk_layernorm_drop_bwd", P(xd), P(rd), P(gd), P(stats), P(dyd), p, P(rng), 5, P(dx), P(dres), P(dgb[0]), P(dgb[1]),
                  rows, C)
        return [y.cpu(), stats.cpu(), dx.cpu(), dres.cpu(), dgb.cpu()]

    y, stats, dx, dres, dgb = twice(run)
    inv = float(torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(p, dtype=torch.float32)))
    assert bool((dx != 0).all())
    ratio = dres / dx                                                # = mask / (1 - p), recovered from the kernel's own outputs
    m = torch.where(ratio.abs() > 0.5, inv, 0.0)
    assert float((ratio - m).abs().max()) <= 1e-6 * inv
    n = m.numel()                                                    # drop fraction within 4 sigma of p (threshold p * 65536)
    assert abs(float((m == 0).float().mean()) - p) < 4 * (p * (1 - p) / n) ** 0.5 + 2.0 ** -16
    chain = 4 * R.cdiv(C // 4, 32) + R.WARP                          # a lane adds its float4 groups (3 + 1 additions each)
    t = R.ln_input(x, res, m)
    ry, rm, rr = R.layernorm_fwd(t, gamma, beta, 1e-5, chain)
    check(y, ry, f"layernorm_drop_fwd y C={C} rows={rows}")
    check(stats[:, 1], rr, f"layernorm_drop_fwd rstd C={C} rows={rows}")
    rdx, rdg, rdb = R.layernorm_bwd(t, gamma, stats[:, 0], stats[:, 1], dy, chain, R.ln_param_chain(rows))
    check(dx, rdx, f"layernorm_drop_bwd dx C={C} rows={rows}")
    check(dres, rdx * R.E(m.double()), f"layernorm_drop_bwd dres C={C} rows={rows}")
    pc = R.ln_param_chain(rows) * R.U32
    check(dgb[0], R.E(rdg.v + base[0].double(), rdg.e + pc * base[0].double().abs()), f"layernorm_drop_bwd dgamma C={C}")
    check(dgb[1], R.E(rdb.v + base[1].double(), rdb.e + pc * base[1].double().abs()), f"layernorm_drop_bwd dbeta C={C}")


# ---- column sums ----------------------------------------------------------------------------------------------------------
# rpb = max(64, ceil(rows / ceil(1056 / ceil(n / 32)))): 63 / 65 rows are one block / two blocks of 64; 200,000 rows of 33
# columns make 528 blocks of 379 rows (rpb >= 64 over many row blocks); n = 31 / 33 / 1024 leave or fill the 32-column tail.
COLSUM = [(1, 1, 1, 0), (63, 31, 40, 1), (65, 33, 33, 0), (200_000, 33, 36, 1), (3000, 1024, 1027, 0), (65, 1, 5, 1)]


@pytest.mark.parametrize("rows,n,ld,acc", COLSUM, ids=[f"rows{a}-n{b}-ld{c}-acc{d}" for a, b, c, d in COLSUM])
def test_colsum(ops, rows, n, ld, acc):
    x = torch.randn(rows, n, generator=_gen(rows + n))
    base = torch.randn(n, generator=_gen(n)) if acc else torch.zeros(n)

    def run():
        out = output(1, n, n + 3)
        if acc:
            out[0, :n] = base.to(DEV)
        ops._call("evk_colsum", P(operand(x, ld)), rows, n, ld, P(out), acc)
        return [body(out, n, "colsum")[0]]

    got, = twice(run)
    assert R.colsum_geometry(200_000, 33) == (379, 528)
    ref = R.esum(R.E(torch.cat([x, base[None]]).double()), 0, R.colsum_chain(rows, n))
    check(got, ref, f"colsum rows={rows} n={n} acc={acc}")


# ---- element-wise -----------------------------------------------------------------------------------------------------------
# small: B = 3 items of T = 37 frames, C = 45 (ragged, lens 0, 1, T - 1, T over the items).  large: rows * C = 1,400 * 800
# = 1,120,000 > 132 * 32 * 256 = 1,081,344, so grid1d's grid-stride loop takes a second trip.
EW_SIZES = {"small": (4, 37, 45, [0, 1, 36, 37]), "large": (2, 700, 800, [700, 699])}


def ew_values(rows, C, seed):
    """inputs spanning softplusf_'s switch at 20 and saturating tanh / sigmoid"""
    g = _gen(seed)
    x = 3 * torch.randn(rows, C, generator=g)
    special = torch.tensor([20.0, 19.999998, 20.000002, -20.0, 25.0, 15.0, -15.0, 40.0, -40.0, 0.0, 1e-6, -1e-6])
    x.view(-1)[:special.numel()] = special
    x.view(-1)[-special.numel():] = special
    return x


@pytest.mark.parametrize("size", list(EW_SIZES))
def test_unary(ops, size):
    B, T, C, _ = EW_SIZES[size]
    rows = B * T
    x = ew_values(rows, C, 1)
    dy = torch.randn(rows, C, generator=_gen(2))
    for op, alpha in ((0, 0.37), (1, 0.1), (2, 0.0), (3, 0.0), (4, 0.0), (6, 0.0)):
        def run():
            y = output(rows, C, C + 2)
            ops._call("evk_unary", op, alpha, P(operand(x, C + 3)), C + 3, P(y), C + 2, rows, C)
            return [body(y, C, "unary")]
        check(twice(run)[0], R.unary(op, alpha, x), f"unary op={op} {size}")
    for op, alpha in ((0, 0.37), (1, 0.1), (2, 0.0), (3, 0.0), (4, 0.0), (5, 0.0)):
        xin = torch.tanh(x) if op == 5 else x                       # op 5: the derivative from the output y = tanh(x)

        def run():
            dx = output(rows, C, C + 1)
            ops._call("evk_unary_bwd", op, alpha, P(operand(xin, C + 3)), C + 3, P(operand(dy, C + 2)), C + 2, P(dx), C + 1, rows, C)
            return [body(dx, C, "unary_bwd")]
        check(twice(run)[0], R.unary_bwd(op, alpha, xin, dy), f"unary_bwd op={op} {size}")


def _len(lens):
    return torch.tensor(lens, dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("size", list(EW_SIZES))
def test_axpby_add_bvec_rowmask_flip(ops, size):
    B, T, C, lens = EW_SIZES[size]
    rows = B * T
    g = _gen(5)
    a, b, c = (torch.randn(rows, C, generator=g) for _ in range(3))
    v = torch.randn(B, C, generator=g)
    keep = R.time_mask(B, T, lens)[:, None]

    def run():
        y = output(rows, C, C + 1)
        ops._call("evk_axpby", P(operand(a, C + 2)), C + 2, 0.5, P(operand(b, C + 3)), C + 3, -1.25, P(operand(c, C + 4)), C + 4, 3.0,
                  P(y), C + 1, rows, C, P(_len(lens)), T)
        y2 = output(rows, C, C + 1)
        ops._call("evk_add_bvec", P(operand(a, C + 2)), C + 2, P(operand(v, C + 5)), C + 5, P(y2), C + 1, B, T, C)
        y3 = output(rows, C, C + 1)
        ops._call("evk_rowmask", P(operand(a, C + 2)), C + 2, P(y3), C + 1, B, T, C, P(_len(lens)))
        y4 = output(rows, C, C + 1)
        ops._call("evk_flip_channels", P(operand(a, C + 2)), C + 2, P(y4), C + 1, rows, C)
        return [body(t, C, "ew") for t in (y, y2, y3, y4)]

    y, y2, y3, y4 = twice(run)
    ref = (0.5 * R.E(a.double()) + (-1.25) * R.E(b.double()) + 3.0 * R.E(c.double()))
    check(y, ref.where(keep.expand(rows, C), R.E(torch.zeros(rows, C))), f"axpby +len {size}")
    check(y2, R.E(a.double()) + R.E(v.double().repeat_interleave(T, 0)), f"add_bvec {size}")
    check(y3, torch.where(keep, a, 0.0), f"rowmask {size}", exact=True)
    check(y4, a.flip(-1), f"flip_channels {size}", exact=True)


@pytest.mark.parametrize("size", list(EW_SIZES))
@pytest.mark.parametrize("with_g", [True, False])
def test_wn_gate_glu_res(ops, size, with_g):
    B, T, H, _ = EW_SIZES[size]
    rows = B * T
    a = ew_values(rows, 2 * H, 7)
    gc = torch.randn(B, 2 * H, generator=_gen(8))
    dact = torch.randn(rows, H, generator=_gen(9))
    xres = torch.randn(rows, H, generator=_gen(10))

    def run():
        acts = output(rows, H, H + 3)
        gd = operand(gc, 2 * H + 1) if with_g else None
        ops._call("evk_wn_gate", P(operand(a, 2 * H + 2)), 2 * H + 2, P(gd), 2 * H + 1, P(acts), H + 3, B, T, H)
        da = output(rows, 2 * H, 2 * H + 1)
        ops._call("evk_wn_gate_bwd", P(operand(a, 2 * H + 2)), 2 * H + 2, P(gd), 2 * H + 1, P(operand(dact, H + 2)), H + 2, P(da),
                  2 * H + 1, B, T, H)
        y = output(rows, H, H + 1)
        xd = operand(xres, H + 4) if with_g else None               # glu_res with x and with x = null
        ops._call("evk_glu_res", P(xd), H + 4, P(operand(a, 2 * H + 2)), 2 * H + 2, P(y), H + 1, rows, H)
        dh = output(rows, 2 * H, 2 * H + 3)
        ops._call("evk_glu_res_bwd", P(operand(a, 2 * H + 2)), 2 * H + 2, P(operand(dact, H + 2)), H + 2, P(dh), 2 * H + 3, rows, H)
        return [body(acts, H, "wn_gate"), body(da, 2 * H, "wn_gate_bwd"), body(y, H, "glu_res"), body(dh, 2 * H, "glu_res_bwd")]

    acts, da, y, dh = twice(run)
    A = R.E(a.double())
    if with_g:
        A = A + R.E(gc.double().repeat_interleave(T, 0))
    ta, sa = A[:, :H], A[:, H:]
    check(acts, R.wn_gate(ta, sa), f"wn_gate g={with_g} {size}")
    d1, d2 = R.wn_gate_bwd(ta, sa, R.E(dact.double()))
    check(da[:, :H], d1, f"wn_gate_bwd tanh half g={with_g} {size}")
    check(da[:, H:], d2, f"wn_gate_bwd sigmoid half g={with_g} {size}")
    check(y, R.glu_res(xres if with_g else None, a[:, :H], a[:, H:]), f"glu_res x={with_g} {size}")
    e1, e2 = R.glu_res_bwd(a[:, :H], a[:, H:], dact)
    check(dh[:, :H], e1, f"glu_res_bwd {size}")
    check(dh[:, H:], e2, f"glu_res_bwd {size}")


@pytest.mark.parametrize("size", list(EW_SIZES))
def test_reparam(ops, size):
    B, T, C, lens = EW_SIZES[size]
    rows = B * T
    g = _gen(12)
    st = torch.cat([torch.randn(rows, C, generator=g), torch.rand(rows, C, generator=g) * 6 - 4], 1)   # logs in [-4, 2]
    nz, dz = torch.randn(rows, C, generator=g), torch.randn(rows, C, generator=g)
    keep = R.time_mask(B, T, lens)[:, None].expand(rows, C)

    def run():
        z = output(rows, C, C + 1)
        ops._call("evk_reparam", P(operand(st, 2 * C + 3)), 2 * C + 3, P(operand(nz, C + 2)), C + 2, P(z), C + 1, B, T, C, P(_len(lens)))
        ds = output(rows, 2 * C, 2 * C + 1)
        ops._call("evk_reparam_bwd", P(operand(st, 2 * C + 3)), 2 * C + 3, P(operand(nz, C + 2)), C + 2, P(operand(dz, C + 4)), C + 4,
                  P(ds), 2 * C + 1, B, T, C, P(_len(lens)))
        return [body(z, C, "reparam"), body(ds, 2 * C, "reparam_bwd")]

    z, ds = twice(run)
    zero = R.E(torch.zeros(rows, C))
    e = R.fast_expf(R.E(st[:, C:].double()))
    check(z, (R.E(st[:, :C].double()) + R.E(nz.double()) * e).where(keep, zero), f"reparam {size}")
    check(ds[:, :C], torch.where(keep, dz, 0.0), f"reparam_bwd dm {size}", exact=True)
    check(ds[:, C:], (R.E(dz.double()) * R.E(nz.double()) * e).where(keep, zero), f"reparam_bwd dlogs {size}")


@pytest.mark.parametrize("size", list(EW_SIZES))
def test_slice_rows_reflect_pad_transposes(ops, size):
    B, T, C, _ = EW_SIZES[size]
    g = _gen(14)
    x = torch.randn(B * T, C, generator=g)
    seg, mul = T // 3, 1
    ids = torch.tensor([0, T - seg, 5, 1][:B], dtype=torch.int64)
    src = torch.cat([b * T + int(ids[b]) * mul + torch.arange(seg) for b in range(B)])
    ynew = torch.randn(B * seg, C, generator=g)
    Tp = T + T // 2
    w = torch.randn(B, T, generator=g)
    dyp = torch.randn(B, Tp, generator=g)
    shift = 3

    def run():
        y = output(B * seg, C, C + 2)
        xd = operand(x, C + 3)
        idd = ids.to(DEV)
        ops._call("evk_slice_rows", P(xd), C + 3, T, P(idd), mul, P(y), C + 2, B, seg, C, 0)
        ops._call("evk_slice_rows", P(xd), C + 3, T, P(idd), mul, P(operand(ynew, C + 2)), C + 2, B, seg, C, 1)   # scatter into x
        pad = torch.full((B, Tp), NAN, device=DEV)
        ops._call("evk_reflect_pad_right", P(w.to(DEV)), T, P(pad), Tp, B, 0)
        adj = torch.full((B, T), NAN, device=DEV)
        ops._call("evk_reflect_pad_right", P(adj), T, P(dyp.to(DEV)), Tp, B, 1)
        ct = torch.full((B, C, T), NAN, device=DEV)                  # [B][T][ld] -> [B][C][T]
        ops._call("evk_transpose_bct_btc", P(operand(x, C + 3)), P(ct), B, C, T, C + 3, 0)
        tc = output(B * T, C, C + 5)                                 # and back: [B][C][T] -> [B][T][ld]
        ops._call("evk_transpose_bct_btc", P(ct), P(tc), B, C, T, C + 5, 1)
        ldy = T + shift + 2
        tr = torch.full((B * C, ldy), SENTINEL, device=DEV)
        tr[:, :T + shift] = NAN
        ops._call("evk_transpose_rows", P(operand(x, C + 3)), C + 3, T * (C + 3), P(tr), ldy, C * ldy, B, T, C, shift)
        xs = xd.cpu()
        assert bool(torch.isnan(xs[:, C:]).all())                    # the scatter writes valid columns only
        return [body(y, C, "slice_rows"), xs[:, :C], pad.cpu(), adj.cpu(), ct.cpu(), body(tc, C, "transpose"),
                body(tr, T + shift, "transpose_rows")]

    y, xs, pad, adj, ct, tc, tr = twice(run)
    check(y, x[src], f"slice_rows gather {size}", exact=True)
    want = x.clone()
    want[src] = ynew
    check(xs, want, f"slice_rows scatter {size}", exact=True)
    s = torch.arange(Tp)
    s = torch.where(s < T, s, 2 * (T - 1) - s)
    check(pad, w[:, s], f"reflect_pad_right {size}", exact=True)
    m = 2 * (T - 1) - torch.arange(T)
    inside = (m >= T) & (m < Tp)
    ref = R.E(dyp[:, :T].double()) + R.E(torch.where(inside, dyp[:, m.clamp(0, Tp - 1)], 0.0).double())
    check(adj, ref, f"reflect_pad_right adjoint {size}")
    xb = x.view(B, T, C)
    check(ct, xb.transpose(1, 2), f"transpose_bct_btc to_bct {size}", exact=True)
    check(tc, x, f"transpose_bct_btc to_btc {size}", exact=True)
    want = torch.zeros(B, C, T + shift)
    want[:, :, shift:] = xb.transpose(1, 2)
    check(tr, want.reshape(B * C, T + shift), f"transpose_rows shift={shift} {size}", exact=True)


# ---- embeddings -------------------------------------------------------------------------------------------------------------
# The backward adds chunks of 256 rows: 1 row, 256 (one full chunk), 257 (a second chunk of one row), 20,000 (79 chunks).
# V * C = 1025 * 512 = 524,800 outputs > 67,584 per ordered_sum trip.
EMB = [(732, 1), (732, 257), (1025, 256), (1025, 20000)]


@pytest.mark.parametrize("V,rows", EMB, ids=[f"V{v}-rows{r}" for v, r in EMB])
def test_embedding(ops, V, rows):
    C = 512
    g = _gen(V + rows)
    tab = torch.randn(V, C, generator=g)
    idx = torch.randint(0, V, (rows,), generator=g)
    hot = [0, 3, 255, 256, rows - 1]                                 # one index repeated within and across 256-row chunks
    idx[[h for h in hot if h < rows]] = 7
    idx[-1] = V - 1 if rows > 1 else idx[-1]
    dy = torch.randn(rows, C, generator=g)
    base = torch.randn(V, C, generator=_gen(1))

    def run():
        idd = idx.to(DEV)
        y = output(rows * 2, C, C + 1)                               # rep = 2: nearest-neighbour upsampling along time
        ops._call("evk_embedding", P(operand(tab, C + 3)), C + 3, P(idd), rows * 2, 2, P(y), C + 1, C)
        dt = output(V, C, C + 3, 0.0)
        dt[:, :C] = base.to(DEV)
        ops._call("evk_embedding_bwd", P(operand(dy, C + 2)), C + 2, P(idd), rows, P(dt), C + 3, C, V)
        return [body(y, C, "embedding"), body(dt, C, "embedding_bwd")]

    # the forward's rows index idx[r // rep]: with rep = 2 it reads idx[0 .. rows - 1] for 2 * rows output rows
    y, dt = twice(run)
    check(y, tab[idx.repeat_interleave(2)], f"embedding V={V} rows={rows}", exact=True)
    chain = min(256, rows) + R.os_chain(R.cdiv(rows, 256))
    v = base.double().index_add(0, idx, dy.double())
    e = chain * R.U32 * base.double().abs().index_add(0, idx, dy.double().abs())
    check(dt, R.E(v, e), f"embedding_bwd V={V} rows={rows}")


# ---- masked mean ------------------------------------------------------------------------------------------------------------
def test_masked_mean(ops):
    """lens: 1, T, > T (clipped to T), a C tail (45 = 32 + 13) and len = 0.  MelStyleEncoder.temporal_avg_pool, the reference
    at this call site, divides the masked sum by the count of valid frames: 0 / 0 = NaN for an empty item in the forward, and
    its backward (masked_fill) gives that item exact zeros.  The kernel does the same, and the test pins it."""
    B, T, C = 5, 50, 45
    lens = [1, 50, 70, 17, 0]
    x = torch.randn(B * T, C, generator=_gen(21))
    dy = torch.randn(B, C, generator=_gen(22))

    def run():
        y = output(B, C, C + 2, 777.0)                               # not NaN: the len = 0 row must come back NaN
        ops._call("evk_masked_mean", P(operand(x, C + 3)), C + 3, P(y), C + 2, B, T, C, P(_len(lens)), 0)
        dx = output(B * T, C, C + 1)
        ops._call("evk_masked_mean", P(dx), C + 1, P(operand(dy, C + 4)), C + 4, B, T, C, P(_len(lens)), 1)
        return [body(y, C, "masked_mean"), body(dx, C, "masked_mean bwd")]

    y, dx = twice(run)
    xb = x.view(B, T, C)
    for b, n in enumerate(lens):
        n = min(n, T)
        if n == 0:
            assert bool(torch.isnan(y[b]).all())
            assert bool((dx.view(B, T, C)[b] == 0).all())
            continue
        ref = R.esum(R.E(xb[b, :n].double()), 0, R.cdiv(n, 8) + 8) / float(n)
        check(y[b], ref, f"masked_mean fwd len={lens[b]}")
        gb = R.E(dy[b].double()) / float(n)
        got = dx.view(B, T, C)[b]
        check(got[:n], row_E(R.E(gb.v[None], gb.e[None]), n), f"masked_mean bwd len={lens[b]}")
        check(got[n:], torch.zeros(T - n, C), "masked_mean bwd beyond len", exact=True)


# ---- sinusoidal position add --------------------------------------------------------------------------------------------
def test_sinepos(ops):
    """B * T * D / 4 = 3 * 400 * 1024 / 4 = 307,200 > 270,336 (the add's grid cap, 1,056 blocks of 256) and B * T * D =
    1,228,800 > 135,168 (the backward's, 528 blocks); batch strides (T + 5) * ldx and (T + 3) * ldy, not T * ld."""
    B, T, D = 3, 400, 1024
    ldx, ldpe, ldy = D + 8, D + 4, D + 12
    xsb, ysb = (T + 5) * ldx, (T + 3) * ldy
    g = _gen(23)
    x, pe, dy = torch.randn(B, T, D, generator=g), torch.randn(T, D, generator=g), torch.randn(B, T, D, generator=g)
    alpha, base = 1.3, 0.25

    def run():
        xd = torch.full((B, T + 5, ldx), NAN)
        xd[:, :T, :D] = x
        yd = torch.full((B, T + 3, ldy), SENTINEL)
        yd[:, :T, :D] = NAN
        dyd = torch.full((B, T + 3, ldy), NAN)
        dyd[:, :T, :D] = dy
        xd, yd, dyd = xd.to(DEV), yd.to(DEV), dyd.to(DEV)
        ped = operand(pe, ldpe)
        al = torch.tensor([alpha], device=DEV)
        ops._call("evk_sinepos_add", P(xd), ldx, xsb, P(ped), ldpe, P(al), P(yd), ldy, ysb, B, T, D)
        da = torch.tensor([base], device=DEV)
        ops._call("evk_sinepos_bwd", P(dyd), ldy, ysb, P(ped), ldpe, P(da), B, T, D)
        yc = yd.cpu()
        assert bool((yc[:, :T, D:] == SENTINEL).all()) and bool((yc[:, T:] == SENTINEL).all())
        return [yc[:, :T, :D], da.cpu()]

    y, da = twice(run)
    check(y, R.E(x.double()) + float(torch.tensor(alpha, dtype=torch.float32)) * R.E(pe.double()), "sinepos_add")
    terms = R.E(dy.double()) * R.E(pe.double())
    chain = R.grid_reduce_chain(B * T * D, R.SINEPOS_BWD_CAP)
    ref = R.esum(R.E(terms.v.reshape(-1), terms.e.reshape(-1)), 0, chain)
    check(da, R.E((ref.v + base).reshape(1), (ref.e + chain * R.U32 * base).reshape(1)), "sinepos_bwd dalpha")


# ---- cross-entropy, DPO head -----------------------------------------------------------------------------------------------
CE_ROWS = [1, 7, 9, 333, 5000]                                       # 1 .. 5000 rows through ce_finalize's 1024-thread loops


@pytest.mark.parametrize("rows", CE_ROWS)
def test_ce_uncounted(ops, rows):
    """V = 1025 classes in rows of ld = 1028 (NaN padding), logits x 30 (lse needs the max subtracted).  The top-k hit rule:
    a valid row is a hit when FEWER THAN k logits are strictly above the target's.  Targets sit at the row maximum, second
    (inside the top 3), fourth (just outside) and at the ignore index 1024."""
    V, ld, k, ignore = 1025, 1028, 3, 1024
    g = _gen(rows)
    lg = 30 * torch.randn(rows, V, generator=g)
    tgt = torch.randint(0, V, (rows,), generator=g)
    order = lg.argsort(-1, descending=True)
    for r in range(rows):
        tgt[r] = order[r, [0, 1, 3, 2, 500][r % 5]] if r % 7 != 6 else ignore
    rpg = 3 if rows >= 9 else 1
    gs = torch.rand(R.cdiv(rows, rpg), generator=g) + 0.5

    def run():
        lgd, tgd = operand(lg, ld), tgt.to(DEV)
        lse, nll = torch.full((rows,), NAN, device=DEV), torch.full((rows,), NAN, device=DEV)
        flags = torch.full((rows,), 255, dtype=torch.uint8, device=DEV)
        out2 = torch.full((2,), NAN, device=DEV)
        ops._call("evk_ce_fwd", P(lgd), ld, P(tgd), rows, V, k, ignore, None, 1, P(lse), P(nll), P(flags), P(out2))
        dl = output(rows, V, ld)
        ops._call("evk_ce_bwd", P(lgd), ld, P(tgd), P(lse), P(gs.to(DEV)), rpg, None, 1, P(dl), ld, rows, V)
        return [lse.cpu(), nll.cpu(), flags.cpu(), out2.cpu(), body(dl, V, "ce_bwd dlogits")]

    lse, nll, flags, out2, dl = twice(run)
    L = R.E(lg.double())
    mx = lg.max(-1).values.double()
    se = R.esum(R.expf(L - R.E(mx[:, None])), -1, R.ln_row_chain(V))
    rlse = R.E(mx) + R.logf(se)
    rnll = rlse - R.E(lg.gather(1, tgt[:, None])[:, 0].double())
    check(lse, rlse, f"ce_fwd lse rows={rows}")
    check(nll, rnll, f"ce_fwd nll rows={rows}")
    valid = tgt != ignore
    above = (lg > lg.gather(1, tgt[:, None])).sum(-1)
    want = valid.to(torch.uint8) | ((valid & (above < k)).to(torch.uint8) << 1)
    assert torch.equal(flags, want)
    hits, nv = int((want >> 1).sum()), int(valid.sum())
    assert float(out2[1]) == float(torch.tensor(hits, dtype=torch.float32) / max(nv, 1))
    check(out2[:1], R.esum(R.E(rnll.v[None], rnll.e[None]), 1, R.cdiv(rows, 1024) + R.BLOCK), f"ce_finalize loss rows={rows}")
    gsr = gs.double().repeat_interleave(rpg)[:rows, None]
    p = R.expf(L - R.E(lse.double()[:, None]))
    onehot = torch.nn.functional.one_hot(tgt, V).double()
    check(dl, R.E(gsr) * (p - R.E(onehot)), f"ce_bwd rows={rows} rows_per_g={rpg}")


def test_ce_uncounted_topk_tie_rule(ops):
    """An exact tie at the k-th place.  The kernel's rule -- hit when fewer than k logits are strictly above the target --
    does not depend on how ties are broken: a target tied for 3rd place is a hit.  The reference's MulticlassAccuracy(
    top_k=3) takes torch.topk's 3 indices, so on such a tie it counts a hit only when topk happens to pick the target;
    without a tie at the boundary the two agree, which this checks row by row."""
    V, k = 1025, 3
    lg = torch.randn(6, V, generator=_gen(31))
    lg[:, :5] = torch.tensor([9.0, 8.0, 7.0, 7.0, 7.0])              # 3rd place shared by columns 2, 3 and 4
    tgt = torch.tensor([0, 1, 2, 3, 4, 5])
    lgd, tgd = lg.to(DEV), tgt.to(DEV)
    lse, nll = torch.empty(6, device=DEV), torch.empty(6, device=DEV)
    flags, out2 = torch.empty(6, dtype=torch.uint8, device=DEV), torch.empty(2, device=DEV)
    ops._call("evk_ce_fwd", P(lgd), V, P(tgd), 6, V, k, 1024, None, 1, P(lse), P(nll), P(flags), P(out2))
    hit = (flags.cpu() >> 1) & 1
    assert hit.tolist() == [1, 1, 1, 1, 1, 0]                        # all three tied targets are hits
    ref_hit = (lg.topk(k, -1).indices == tgt[:, None]).any(-1)       # MulticlassAccuracy(top_k=3)'s test, per row
    assert hit[[0, 1, 5]].bool().tolist() == ref_hit[[0, 1, 5]].tolist()
    assert int(ref_hit[2:5].sum()) == 1                              # topk keeps one of the three tied columns


def test_dpo_head_uncounted(ops):
    """z = -beta (A - R) of both signs and |z| >= 20 (both softplus branches, sigmoid saturated); sums of 300 / 280 tokens
    through a 256-thread block_sum."""
    B, Yc, Yr, beta = 4, 300, 280, 0.2
    g = _gen(41)
    nc, nr = torch.rand(B, Yc, generator=g) * 4, torch.rand(B, Yr, generator=g) * 4
    nr[0] += 0.75                                                    # z = beta (sc - sr): about -34, +38, 0 and 8 (sums ~ 2 Y)
    nc[1] += 0.5
    nr[2] += 0.14

    def run():
        out3, cc, cr = torch.full((3,), NAN, device=DEV), torch.full((B,), NAN, device=DEV), torch.full((B,), NAN, device=DEV)
        ops._call("evk_dpo_head", P(nc.to(DEV)), Yc, None, P(nr.to(DEV)), Yr, None, B, beta, P(out3), P(cc), P(cr))
        return [out3.cpu(), cc.cpu(), cr.cpu()]

    out3, cc, cr = twice(run)
    bf = float(torch.tensor(beta, dtype=torch.float32))
    sc = R.esum(R.E(nc.double()), 1, R.cdiv(Yc, 256) + R.BLOCK)
    sr = R.esum(R.E(nr.double()), 1, R.cdiv(Yr, 256) + R.BLOCK)
    z = (sc - sr) * bf                                               # -beta ((-sc) - (-sr))
    assert bool((z.v > 20).any()) and bool((z.v < -20).any()) and bool((z.v.abs() < 20).any())
    pos = z.v > 0
    sp_pos = z + R.log1pf(R.expf(-z))
    sp_neg = R.log1pf(R.expf(z))
    sp = sp_pos.where(pos, sp_neg)
    sg = 1.0 / (1.0 + R.expf(-z))
    check(cc, 1.0 + sg * bf / float(B), "dpo_head coef_c")
    check(cr, -(sg * bf) / float(B), "dpo_head coef_r")
    l1, l2 = R.esum(sc, 0, B), R.esum(sp, 0, B)
    l2b = l2 / float(B)
    check(out3, R.E(torch.stack([l1.v, l2b.v, l1.v + l2b.v]), torch.stack([l1.e, l2b.e, l1.e + l2b.e + R.U32 * (l1.v + l2b.v).abs()])),
          "dpo_head out3")


# ---- losses ---------------------------------------------------------------------------------------------------------------
# n = 600,000 > 132 * 16 * 256 = 540,672: the g1 grid-stride loops take a second trip.
@pytest.mark.parametrize("n", [1000, 600_000])
def test_reduce_loss(ops, n):
    g = _gen(n)
    a, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
    b[:7] = a[:7]                                                    # |a - b| = 0: sign 0 in the backward
    scale, base, gout = 0.37, 1.5, 0.8

    def run():
        outs = []
        for kind in (0, 1, 2):
            out = torch.tensor([base], device=DEV)
            ops._call("evk_reduce_loss", kind, P(a.to(DEV)), P(b.to(DEV)), n, scale, P(out))
            da = torch.full((n,), NAN, device=DEV)
            ops._call("evk_reduce_loss_bwd", kind, P(a.to(DEV)), P(b.to(DEV)), n, scale, P(torch.tensor([gout], device=DEV)), P(da))
            outs += [out.cpu(), da.cpu()]
        return outs

    res = twice(run)
    gsc = R.E(torch.tensor(float(torch.tensor(gout, dtype=torch.float32)) * float(torch.tensor(scale, dtype=torch.float32))))
    gsc = R.E(gsc.v, R.U32 * gsc.v.abs())
    A = R.E(a.double())
    for kind in (0, 1, 2):
        ref, G = R.reduce_loss(kind, a, b, float(torch.tensor(scale, dtype=torch.float32)))
        oc = R.os_chain(G) * R.U32
        check(res[2 * kind], R.E((ref.v + base).reshape(1), (ref.e + oc * (ref.v.abs() + base)).reshape(1)), f"reduce_loss kind={kind} n={n}")
        if kind == 0:
            d = -2.0 * (1.0 - A)
        elif kind == 1:
            d = 2.0 * A
        else:
            d = R.E(torch.sign(a.double() - b.double()))
        check(res[2 * kind + 1], gsc * d, f"reduce_loss_bwd kind={kind} n={n}")


def test_kl_loss(ops):
    """B * T * C = 4 * 500 * 300 = 600,000 > 540,672 (a second trip); logs_p in [-7, 3], so __expf(-2 logs_p) reaches e^14 and
    its error 2 + floor(1.173 * 14) = 18 ulp; lens: a full row, a row of 1, 250 and T - 1."""
    B, T, C = 4, 500, 300
    ld = C + 3
    lens = [500, 1, 250, 499]
    g = _gen(51)
    zp, lq, mp = (torch.randn(B * T, C, generator=g) for _ in range(3))
    lp = torch.rand(B * T, C, generator=g) * 10 - 7
    keep = R.time_mask(B, T, lens)[:, None].expand(-1, C)
    gout, gscale, base = 0.5, 0.125, -2.0

    def run():
        dz, dq, dm, dp_ = (output(B * T, C, ld + 1) for _ in range(4))
        out = torch.tensor([base], device=DEV)
        args = [P(operand(zp, ld)), ld, P(operand(lq, ld + 1)), ld + 1, P(operand(mp, ld + 2)), ld + 2, P(operand(lp, ld + 3)), ld + 3, B, T, C,
                P(_len(lens))]
        ops._call("evk_kl_loss", *args, P(out))
        ops._call("evk_kl_loss_bwd", *args, P(torch.tensor([gout], device=DEV)), gscale, P(dz), P(dq), P(dm), P(dp_), ld + 1)
        return [out.cpu()] + [body(t, C, "kl_loss_bwd") for t in (dz, dq, dm, dp_)]

    out, dz, dq, dm, dp_ = twice(run)
    t = R.kl_terms(zp, lq, mp, lp)
    zero = torch.zeros_like(t.v)
    chain = R.grid_reduce_chain(B * T * C, R.G1_CAP)
    tv, te = torch.where(keep, t.v, zero), torch.where(keep, t.e, zero)
    check(out, R.E((tv.sum() + base).reshape(1), (te.sum() + chain * R.U32 * (tv.abs().sum() + abs(base))).reshape(1)), "kl_loss")
    a, am, q, p = R.kl_bwd(zp, lq, mp, lp, gout, gscale)
    Z = R.E(zero)
    check(dz, a.where(keep, Z), "kl_loss_bwd dz_p")
    check(dm, am.where(keep, Z), "kl_loss_bwd dm_p")
    check(dq, q.where(keep, Z), "kl_loss_bwd dlogs_q")
    check(dp_, p.where(keep, Z), "kl_loss_bwd dlogs_p")


# ---- AdamW ------------------------------------------------------------------------------------------------------------------
def test_adamw(ops):
    """n = 600,000 past the grid cap; steps 1-3 through the device step counter (hyper[1] advanced by evk_scalar_add, as the
    stage-2 step does); grad_scale, lr_scale and weight decay != 0; the gnorm_sq partials."""
    n = 600_000
    g = _gen(61)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) for _ in range(3)]
    hp = dict(lr=2e-4, lr_scale=0.5, b1=0.8, b2=0.99, eps=1e-9, wd=0.01, grad_scale=0.25)

    def run():
        p, m, v = p0.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        hyper = torch.tensor([hp["lr"], 0.0], device=DEV)
        outs = []
        for gr in grads:
            ops.scalar_add(hyper[1:], 1.0)
            gn = torch.zeros(1, device=DEV)
            ops._call("evk_adamw_flat", P(p), P(gr.to(DEV)), P(m), P(v), n, P(hyper), hp["lr_scale"], hp["b1"], hp["b2"], hp["eps"], hp["wd"],
                      hp["grad_scale"], P(gn))
            outs += [p.cpu(), m.cpu(), v.cpu(), gn.cpu()]
        return outs

    res = twice(run)
    P_, M, V = R.E(p0.double()), R.E(torch.zeros(n)), R.E(torch.zeros(n))
    chain = R.grid_reduce_chain(n, R.G1_CAP)
    for s, gr in enumerate(grads):
        P_, M, V, GG = R.adamw_step(P_, gr, M, V, step=s + 1, **hp)
        p, m, v, gn = res[4 * s:4 * s + 4]
        check(p, P_, f"adamw p step {s + 1}")
        check(m, M, f"adamw m step {s + 1}")
        check(v, V, f"adamw v step {s + 1}")
        check(gn, R.E(GG.v.sum().reshape(1), (GG.e.sum() + chain * R.U32 * GG.v.sum()).reshape(1)), f"adamw gnorm_sq step {s + 1}")
