"""Every output of the tensor-core contraction kernels, checked bit for bit with exactly representable operands.

The operands are small integers (tests/exact_ref.py says why every product and partial sum is then exact), so with the
truncation compensation off each kernel must reproduce the float64 result exactly at every output: a wrong tile-edge
predicate, a dropped K block or split, a tap shift into the wrong residue copy or a misplaced float4 of the epilogue
changes an output by a whole unit.  A whole-tensor relative-L2 gate cannot see one such output among millions.

Kernels: gemm_tma_kernel (evk_gemm_tf32, the flat Linear path, tap-sum and phased strided convs), conv_wgrad_kernel,
gconv_tc_kernel, the mma.sync and direct fallbacks, and both kernels of evk_conv2d_fwd.  Every case asserts from
the library's dispatch accounting that its flops went to the kernel family it is about.
"""
import math

import pytest
import torch

from tests import exact_ref as R
from tests.test_gpu_uvr5 import CONV_GRID
from tests.test_gpu_uvr5_echo import CONV_HW_GRID

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
TRUNC_COMP = 3.52e-4                   # the library's default compensation per truncated operand
FWD = ("fwd_gemm_tma", "fwd_gconv_tc", "fwd_mma_sync", "fwd_direct", "fwd_gemv")
WGRAD = ("wgrad_gemm_tma", "wgrad_mma_sync", "wgrad_direct")
NAN = float("nan")


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    L = lib.init()
    L.evk_set_precise(0)
    try:
        yield ops
    finally:
        L.evk_set_precise(0)
        L.evk_set_tma_options(1, 1, TRUNC_COMP)
        L.evk_set_backend(1)
        L.evk_set_backend_tma(1)


@pytest.fixture(autouse=True)
def exact_mode(ops):
    """compensation off, default dispatch; restored whatever the test did"""
    from easevoice_trainer_b200 import lib
    L = lib.init()
    L.evk_set_tma_options(1, 1, 0.0)
    yield L
    L.evk_set_precise(0)
    L.evk_set_backend(1)
    L.evk_set_backend_tma(1)
    L.evk_set_tma_options(1, 1, TRUNC_COMP)


def _bn(n):
    return 128 if n > 64 else (64 if n > 32 else 32)


def assert_exact(got, ref, what, axes, tiles=None):
    """got == ref at every element.  axes names the dimensions; tiles maps an axis to the tile size it is cut into, so
    the report shows (index, tile) for the first mismatches."""
    got, ref = got.detach().double().to(ref.device), ref.detach().double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    bad = ~(got == ref)
    n = int(bad.sum())
    if n:
        lines = []
        for idx in bad.nonzero()[:6].tolist():
            coord = ", ".join(f"{a}={i}" + (f" (tile {i // tiles[a]})" if tiles and a in tiles else "") for a, i in zip(axes, idx))
            lines.append(f"  [{coord}] got {float(got[tuple(idx)])!r} want {float(ref[tuple(idx)])!r}")
        pytest.fail(f"{what}: {n} of {bad.numel()} outputs differ from the exact result\n" + "\n".join(lines))


def assert_family(ops, fam, slots, what):
    st = ops.dispatch_stats()
    others = {k: st[k] for k in slots if k != fam and st[k]}
    assert st[fam] > 0 and not others, f"{what}: expected the flops on {fam}, dispatch accounting says {st}"


def assert_bound(value, what):
    assert value <= R.EXACT_BOUND, f"{what}: sum |a||b| = {value} > 2^20, the integers would not stay exact"


# ---- evk_gemm_tf32 ----------------------------------------------------------------------------------------------------
def _gemm_ref(a, b, bias, res, epi):
    ref = a.to(DEV) @ b.to(DEV).t()
    if epi != "none":
        ref = ref + bias.to(DEV)
    if epi == "brr":
        ref = torch.relu(ref + res.to(DEV))
    elif epi == "lrelu":
        ref = R.act_ref(ref, R.ACT_LRELU)
    return ref


def _padded(t, extra=4, fill=NAN):
    """t [rows, K] on the device as a column slice of a buffer whose pitch padding holds `fill`"""
    buf = torch.full((t.shape[0], t.shape[1] + extra + (-t.shape[1]) % 4), fill, device=DEV)
    buf[:, :t.shape[1]] = t.to(DEV)
    return buf[:, :t.shape[1]]


# every shape with a plain output; the smaller ones also into an ldd > N view and into one that is not 16-byte aligned
GEMM_RUNS = [(c, "plain") for c in R.GEMM_CASES] + [(c, lay) for c in R.GEMM_CASES if c[0] <= 300 for lay in ("ldd", "offset")]


@pytest.mark.parametrize("case,layout", GEMM_RUNS, ids=[f"M{m}-N{n}-K{k}-{e}-{lay}" for (m, n, k, e), lay in GEMM_RUNS])
def test_gemm_tf32(ops, case, layout):
    M, N, K, epi = case
    g = torch.Generator().manual_seed(M * 7 + N * 13 + K)
    a, b = R.ints((M, K), R.RX, g), R.ints((N, K), R.RW, g)
    bias, res = R.ints((N,), R.RB, g), R.ints((M, N), R.RB, g)
    assert_bound(R.gemm_case_bound(K), "gemm")
    ad, bd = _padded(a), _padded(b)                      # K-pitch padding of NaN: not part of the operands
    SENT = -12345.0
    if layout == "plain":
        obuf = torch.full((M * N,), SENT, device=DEV)
        out = obuf.view(M, N)
    else:                                                # ldd > N, and (offset) a base that is not 16-byte aligned
        ldd = N + 7
        off = 1 if layout == "offset" else 0
        obuf = torch.full((off + M * ldd,), SENT, device=DEV)
        out = obuf[off:].view(M, ldd)[:, :N]
    resd = _padded(res) if epi == "brr" else None
    ops.dispatch_reset()
    act = {"none": ops.ACT_NONE, "brr": ops.ACT_RELU, "lrelu": ops.ACT_LRELU}[epi]
    ops.gemm_tf32(ad, bd, out=out, bias=bias.float().to(DEV) if epi != "none" else None, res=resd, act=act, slope=R.LRELU_SLOPE)
    torch.cuda.synchronize()
    assert_family(ops, "gemm_tf32", FWD + WGRAD + ("gemm_tf32",), "gemm_tf32")
    assert_exact(out, _gemm_ref(a, b, bias, res, epi), f"gemm_tf32 M{M} N{N} K{K} {epi} {layout}", ("m", "n"),
                 {"m": 128, "n": _bn(N)})
    written = torch.zeros_like(obuf, dtype=torch.bool)
    if layout == "plain":
        written[:] = True
    else:
        written[off:].view(M, ldd)[:, :N] = True
    assert (obuf[~written] == SENT).all(), "gemm_tf32 wrote outside its output view"


@pytest.mark.parametrize("case", R.SPLITK_CASES, ids=[f"M{m}-N{n}-K{k}-s{s}" for m, n, k, s in R.SPLITK_CASES])
def test_gemm_tf32_split_k(ops, case):
    M, N, K, splits = case
    g = torch.Generator().manual_seed(M + N + K + splits)
    a, b = R.ints((M, K), 1, g), R.ints((N, K), 1, g)
    init = R.ints((M, N), 100, g)
    assert_bound(R.gemm_case_bound(K, 1, 1), "split-K gemm")
    out = init.float().to(DEV)
    ops.dispatch_reset()
    ops.gemm_tf32(_padded(a), _padded(b), out=out, splits=splits)
    torch.cuda.synchronize()
    assert_family(ops, "gemm_tf32", FWD + WGRAD + ("gemm_tf32",), "split-K gemm_tf32")
    assert_exact(out, init.to(DEV) + a.to(DEV) @ b.to(DEV).t(), f"split-K gemm M{M} N{N} K{K} splits {splits}", ("m", "n"),
                 {"m": 128, "n": _bn(N)})


# ---- Linear on the flat GEMM path ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", R.LINEAR_CASES, ids=[f"B{b}-T{t}-C{c}-N{n}-{e}" for b, t, c, n, e in R.LINEAR_CASES])
def test_linear_flat(ops, case):
    B, T, C, N, epi = case
    g = torch.Generator().manual_seed(B * 1000 + T + C + N)
    x, w = R.ints((B, T, C), R.RX, g), R.ints((N, C), R.RW, g)
    bias, res = R.ints((N,), R.RB, g), R.ints((B, T, N), R.RB, g)
    assert_bound(R.gemm_case_bound(C), "linear")
    xbuf = torch.full((B, T, C + 4), NAN, device=DEV)
    xbuf[..., :C] = x.to(DEV)
    act = {"none": ops.ACT_NONE, "brr": ops.ACT_RELU, "lrelu": ops.ACT_LRELU}[epi]
    with torch.no_grad():
        pw = ops.pack_weight(w.float().to(DEV).unsqueeze(-1))
        ops.dispatch_reset()
        y = ops.linear(xbuf[..., :C], pw, bias.float().to(DEV) if epi != "none" else None, act=act, slope=R.LRELU_SLOPE,
                       res=res.float().to(DEV) if epi == "brr" else None)
        torch.cuda.synchronize()
    assert_family(ops, "fwd_gemm_tma", FWD, "linear")
    ref = _gemm_ref(x.reshape(-1, C), w, bias, res.reshape(-1, N), epi).reshape(B, T, N)
    assert_exact(y, ref, f"linear B{B} T{T} C{C} N{N} {epi}", ("b", "t", "n"), {"n": _bn(N)})


# the dropout of a Linear on every route of evk_gconv_fwd: route name -> dispatch slot
DROP_ROUTES = {"tma": "fwd_gemm_tma", "gconv_tc": "fwd_gconv_tc", "mma_sync": "fwd_mma_sync", "precise": "fwd_mma_sync",
               "direct": "fwd_direct"}


def _dropout_linear(ops, L, route):
    """-> (y, 2 relu(pre)) of linear + ReLU + dropout(0.5) with the same seed and tag, on the given route"""
    B, T, C, N = 2, 1000, 64, 96
    g = torch.Generator().manual_seed(5)
    x, w, bias = R.ints((B, T, C), R.RX, g), R.ints((N, C), R.RW, g), R.ints((N,), R.RB, g)
    xd = x.float().to(DEV)
    if route == "direct":                                # x one float into its buffer: not 16-byte aligned
        buf = torch.empty(xd.numel() + 1, device=DEV)
        buf[1:] = xd.flatten()
        xd = buf[1:].view(B, T, C)
    {"gconv_tc": lambda: L.evk_set_backend_tma(0), "mma_sync": lambda: L.evk_set_backend(0),
     "precise": lambda: L.evk_set_precise(1)}.get(route, lambda: None)()
    try:
        with torch.no_grad():
            pw = ops.pack_weight(w.float().to(DEV).unsqueeze(-1))
            ops.manual_seed(11)
            ops.dispatch_reset()
            y = ops.linear(xd, pw, bias.float().to(DEV), act=ops.ACT_RELU, drop=(0.5, "exact-dropout"))
            torch.cuda.synchronize()
    finally:
        L.evk_set_precise(0)
        L.evk_set_backend(1)
        L.evk_set_backend_tma(1)
    keep = 2.0 * torch.relu(x.reshape(-1, C).to(DEV) @ w.to(DEV).t() + bias.to(DEV)).reshape(B, T, N)
    return y.double(), keep


def test_linear_fused_dropout(ops):
    """the DROP instantiation of the fast epilogue: every output is 0 or exactly 2 relu(pre) at p = 0.5"""
    B, T, C, N = 2, 1000, 64, 96
    g = torch.Generator().manual_seed(5)
    x, w, bias = R.ints((B, T, C), R.RX, g), R.ints((N, C), R.RW, g), R.ints((N,), R.RB, g)
    with torch.no_grad():
        pw = ops.pack_weight(w.float().to(DEV).unsqueeze(-1))
        ops.manual_seed(11)
        ops.dispatch_reset()
        y = ops.linear(x.float().to(DEV), pw, bias.float().to(DEV), act=ops.ACT_RELU, drop=(0.5, "exact-dropout"))
        torch.cuda.synchronize()
    assert_family(ops, "fwd_gemm_tma", FWD, "fused dropout linear")
    keep = 2.0 * torch.relu(x.reshape(-1, C).to(DEV) @ w.to(DEV).t() + bias.to(DEV)).reshape(B, T, N)
    y = y.double()
    ok = (y == 0) | (y == keep)
    assert ok.all(), f"{int((~ok).sum())} outputs are neither dropped nor 2 relu(pre); first at {(~ok).nonzero()[0].tolist()}"
    live = keep > 0
    frac = float((y[live] != 0).double().mean())
    assert 0.45 < frac < 0.55, frac


@pytest.mark.parametrize("route", [r for r in DROP_ROUTES if r != "tma"])
def test_linear_dropout_pass(ops, exact_mode, route):
    """the routes whose epilogue has no dropout: the pass after the launch leaves every output 0 or exactly 2 relu(pre)"""
    y, keep = _dropout_linear(ops, exact_mode, route)
    assert_family(ops, DROP_ROUTES[route], FWD, f"dropout linear on {route}")
    ok = (y == 0) | (y == keep)
    assert ok.all(), f"{int((~ok).sum())} outputs are neither dropped nor 2 relu(pre); first at {(~ok).nonzero()[0].tolist()}"
    live = keep > 0
    frac = float((y[live] != 0).double().mean())
    assert 0.45 < frac < 0.55, frac


def test_linear_dropout_mask_is_the_same_on_every_route(ops, exact_mode):
    """the keep pattern depends on (seed, offset, stream id, output index) only, not on the kernel that computed y"""
    dropped = {}
    for route in DROP_ROUTES:
        y, keep = _dropout_linear(ops, exact_mode, route)
        dropped[route] = (y == 0) & (keep > 0)
    first = dropped["tma"]
    assert first.any()
    for route, d in dropped.items():
        assert torch.equal(d, first), f"{route}: {int((d != first).sum())} positions dropped differently from the TMA epilogue"


def test_dropout_needs_relu(ops):
    """the library rejects dropout after any activation but ReLU (a backward recovers the mask from the saved output)"""
    x = torch.ones(1, 600, 64, device=DEV)
    pw = ops.pack_weight(torch.ones(64, 64, 1, device=DEV))
    y = torch.empty(1, 600, 64, device=DEV)
    with pytest.raises(RuntimeError, match="error -1.*EVK_ACT_RELU"):
        ops._fwd_like(x, 600, pw.pa, pw.pa.shape[2], 64 * pw.pa.shape[2], 64, 64, y, J=600, P=1, is_=1, off=[0],
                      act=ops.ACT_GELU, drop=(0.5, ops.stream_id("exact-dropout")))


# ---- Linear of a few rows: route 0 (evk_gemv_rows) or a TF32 route ---------------------------------------------------------
@pytest.mark.parametrize("case", R.GEMV_CASES, ids=[c[0].replace(" ", "_") for c in R.GEMV_CASES])
def test_linear_skinny_route(ops, case):
    name, B, T, C, N, act, use_res, no_grad, fam = case
    g = torch.Generator().manual_seed(B * 100 + T + C)
    x, w, bias, res = R.ints((B, T, C), R.RX, g), R.ints((N, C), R.RW, g), R.ints((N,), R.RB, g), R.ints((B, T, N), R.RB, g)
    assert_bound(R.gemm_case_bound(C), name)
    with torch.no_grad():
        pw = ops.pack_weight(w.float().to(DEV).unsqueeze(-1))
    with torch.set_grad_enabled(not no_grad):
        ops.dispatch_reset()
        y = ops.linear(x.float().to(DEV), pw, bias.float().to(DEV), act=act, slope=R.LRELU_SLOPE,
                       res=res.float().to(DEV) if use_res else None)
        torch.cuda.synchronize()
    assert_family(ops, fam, FWD, name)
    wr = pw.pa[0, :N, :C].double()                      # the operand the kernels read
    pre = (x.reshape(-1, C).to(DEV) @ wr.t() + bias.to(DEV)).reshape(B, T, N) + (res.to(DEV) if use_res else 0)
    if act == R.ACT_GELU:
        ref = torch.nn.functional.gelu(pre)
        err = float(((y.double() - ref).abs() / (ref.abs() + 1)).max())
        assert err < 1e-6, f"{name}: GELU epilogue off by {err}"
    else:
        assert_exact(y, R.act_ref(pre, act), name, ("b", "t", "n"))


# ---- convolutions through ops.conv --------------------------------------------------------------------------------------
def _lens(B, L):
    return torch.tensor([L] + [max(L - 7 * (b + 1), 3) for b in range(B - 1)])


def _to_cl(t):
    """[B, C, T, P] -> channels-last rows [B, T * P, C]"""
    B, C, T, P = t.shape
    return t.permute(0, 2, 3, 1).reshape(B, T * P, C)


def _run_conv(ops, case, seed, backward=True, comp=0.0):
    """-> list of (what, got, ref, axes, tiles) after running the case and its float64 reference"""
    name, B, Tin, C, N, Q, stride, pad, dil, P, G, act, use_res, masks, ffam, dfam, wfam, (slab, mt2, *mode) = case
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_tma_options(slab, mt2, comp)
    if "precise" in mode:
        lib.init().evk_set_precise(1)
    x0 = 1 if "x+1" in mode else 0
    for what, bnd in zip(("forward", "data gradient", "weight gradient"), R.conv_case_bounds(case)):
        assert_bound(bnd, f"{name} {what}")
    g = torch.Generator().manual_seed(seed)
    J = R.conv_out_len(Tin, Q, stride, pad, dil)
    x, v, bias = R.ints((B, C, Tin, P), R.RX, g), R.ints((N, C // G, Q), R.RW, g), R.ints((N,), R.RB, g)
    res = R.ints((B, N, J, P), R.RB, g) if use_res else None
    gy = R.ints((B, N, J, P), R.RDY, g)
    lens = _lens(B, Tin if masks == "inout" else J) if masks else None

    # float64 reference (unfold + matmul on the device: cuBLAS DGEMM, no TF32 anywhere)
    xr, vr, br = [t.to(DEV).requires_grad_(True) for t in (x, v, bias)]
    resr = res.to(DEV).requires_grad_(True) if use_res else None
    xin = xr
    if masks == "inout":
        xin = xr * (torch.arange(Tin)[None, :] < lens[:, None]).double().to(DEV)[:, None, :, None]
    assert_bound(float(R.conv1d_ref(x.abs().to(DEV), v.abs().to(DEV), None, stride, pad, dil, G).max()), f"{name} forward operands")
    pre = R.conv1d_ref(xin, vr, br, stride, pad, dil, G)
    if use_res:
        pre = pre + resr
    yr = R.act_ref(pre, act)
    if masks:
        yr = yr * (torch.arange(J)[None, :] < lens[:, None]).double().to(DEV)[:, None, :, None]

    # ours: input as a channel slice whose pitch padding is NaN
    xbuf = torch.full((B, Tin * P, C + 4), NAN, device=DEV)
    xbuf[..., x0:x0 + C] = _to_cl(x).to(DEV)
    xbuf.requires_grad_(backward)
    vd, bd = v.float().to(DEV).requires_grad_(backward), bias.float().to(DEV).requires_grad_(backward)
    resd = _to_cl(res).float().to(DEV).requires_grad_(backward) if use_res else None
    ln = lens.to(DEV, torch.int32) if masks else None
    pw = ops.pack_weight(vd)
    ops.dispatch_reset()
    yo = ops.conv(xbuf[..., x0:x0 + C], pw, bd, stride=stride, pad=pad, dil=dil, P=P, groups=G, act=act, slope=R.LRELU_SLOPE, res=resd,
                  in_len=ln if masks == "inout" else None, out_len=ln)
    torch.cuda.synchronize()
    assert_family(ops, ffam, FWD + WGRAD, f"{name} forward")
    out = [("y", yo, _to_cl(yr.detach()), ("b", "row", "n"), {"row": 128, "n": _bn(N)})]
    if not backward:
        return out
    yr.backward(gy.to(DEV))
    ops.dispatch_reset()
    yo.backward(_to_cl(gy).float().to(DEV))
    torch.cuda.synchronize()
    assert_family(ops, wfam, WGRAD, f"{name} weight gradient")
    if dfam:
        assert_family(ops, dfam, FWD, f"{name} data gradient")
    assert (xbuf.grad[..., :x0] == 0).all() and (xbuf.grad[..., x0 + C:] == 0).all()
    out += [("dx", xbuf.grad[..., x0:x0 + C], _to_cl(xr.grad), ("b", "row", "c"), {"row": 128, "c": _bn(C)}),
            ("dW", vd.grad, vr.grad, ("n", "c", "tap"), {"n": 128, "c": 128}),
            ("dbias", bd.grad, br.grad, ("n",), None)]
    if use_res:
        out.append(("dres", resd.grad, _to_cl(resr.grad), ("b", "row", "n"), {"row": 128}))
    return out


@pytest.mark.parametrize("case", R.CONV_CASES, ids=[c[0].replace(" ", "_") for c in R.CONV_CASES])
def test_conv(ops, case):
    for what, got, ref, axes, tiles in _run_conv(ops, case, seed=hash(case[0]) % 10007):
        assert_exact(got, ref, f"conv[{case[0]}] {what}", axes, tiles)


def test_conv_post_tanh(ops):
    """conv_post: 16 -> 1 channel carried as 4 (zero weight rows) with tanh on gconv_tc_kernel"""
    B, T, C, Q, pad = R.CONV_POST
    g = torch.Generator().manual_seed(3)
    x, v, bias = R.ints((B, C, T, 1), R.RX, g), R.ints((1, C, Q), R.RW, g), R.ints((1,), R.RB, g)
    assert_bound(C * Q * R.RX * R.RW, "conv_post")
    with torch.no_grad():
        pw = ops.pack_weight(v.float().to(DEV), pad0=4)
        ops.dispatch_reset()
        y = ops.conv(_to_cl(x).float().to(DEV), pw, torch.nn.functional.pad(bias.float(), (0, 3)).to(DEV), pad=pad,
                     act=ops.ACT_TANH)
        torch.cuda.synchronize()
    assert_family(ops, "fwd_gconv_tc", FWD, "conv_post")
    pre = R.conv1d_ref(x.to(DEV), v.to(DEV), bias.to(DEV), 1, pad, 1)[:, 0, :, 0]
    err = float((y[..., 0].double() - torch.tanh(pre)).abs().max())
    assert err <= 2e-6, err
    assert (y[..., 1:] == 0).all()


@pytest.mark.parametrize("case", R.CONVT_CASES, ids=["-".join([f"{a}-{b}-k{k}-s{s}-T{t}"] + m) for a, b, k, s, t, *m in R.CONVT_CASES])
def test_conv_transpose(ops, case):
    """ConvTranspose1d forward: the os / o0 output mapping of the TMA kernel's epilogue; backward on mma.sync"""
    (Cin, Cout, Q, s, T), mode = case[:5], case[5:]
    x0 = 1 if "x+1" in mode else 0
    pad = (Q - s) // 2
    g = torch.Generator().manual_seed(Cin + Q + T)
    x, v, bias = R.ints((2, Cin, T), R.RX, g), R.ints((Cin, Cout, Q), R.RW, g), R.ints((Cout,), R.RB, g)
    Tout = (T - 1) * s - 2 * pad + Q
    gy = R.ints((2, Cout, Tout), R.RDY, g)
    assert_bound(Cin * math.ceil(Q / s) * R.RX * R.RW, "convT forward")
    assert_bound(2 * T * R.RX * R.RDY, "convT weight gradient")
    xr, vr, br = [t.to(DEV).requires_grad_(True) for t in (x, v, bias)]
    yr = R.conv_transpose1d_ref(xr, vr, br, s, pad)
    yr.backward(gy.to(DEV))
    xbuf = torch.zeros((2, T, x0 + Cin), device=DEV)
    xbuf[..., x0:] = x.transpose(1, 2).to(DEV)
    xbuf.requires_grad_(True)
    vd, bd = v.float().to(DEV).requires_grad_(True), bias.float().to(DEV).requires_grad_(True)
    ops.dispatch_reset()
    yo = ops.conv_transpose(xbuf[..., x0:], ops.pack_weight(vd), bd, stride=s, pad=pad)
    torch.cuda.synchronize()
    assert_family(ops, "fwd_direct" if x0 else "fwd_gemm_tma" if T >= 1000 else "fwd_gconv_tc", FWD, "convT forward")
    ops.dispatch_reset()
    yo.backward(gy.transpose(1, 2).float().to(DEV))
    torch.cuda.synchronize()
    assert_family(ops, "wgrad_direct" if x0 else "wgrad_mma_sync", WGRAD, "convT weight gradient")
    n = f"convT[{Cin}->{Cout} k{Q} s{s} T{T}{' x+1' if x0 else ''}]"
    assert_exact(yo, yr.detach().transpose(1, 2), n + " y", ("b", "t", "n"), {"t": 128, "n": _bn(Cout)})
    assert_exact(xbuf.grad[..., x0:], xr.grad.transpose(1, 2), n + " dx", ("b", "t", "c"), {"t": 128})
    assert_exact(vd.grad, vr.grad, n + " dW", ("ci", "co", "tap"), None)
    assert_exact(bd.grad, br.grad, n + " dbias", ("n",), None)


def test_cross_family_bit_identical(ops, exact_mode):
    """One TMA problem and one gconv_tc problem on every kernel family that can run them: default dispatch, TMA off,
    mma.sync, and 3xTF32.  All outputs are the same bits (and the exact result)."""
    L = exact_mode
    cases = [c for c in R.CONV_CASES if c[0] in ("tma k3 36->96 C tail", "tc resblock k7 d3 c16 +res")]
    assert len(cases) == 2
    for case in cases:
        results = []
        for label, fam, setup in (("default", case[14], lambda: None),
                                  ("tma off", "fwd_gconv_tc", lambda: L.evk_set_backend_tma(0)),
                                  ("mma.sync", "fwd_mma_sync", lambda: L.evk_set_backend(0)),
                                  ("3xTF32", "fwd_mma_sync", lambda: L.evk_set_precise(1))):
            setup()
            try:
                with torch.no_grad():
                    (_, y, ref, axes, tiles), = _run_conv(ops, case[:14] + (fam,) + case[15:], seed=17, backward=False)
            finally:
                L.evk_set_precise(0); L.evk_set_backend(1); L.evk_set_backend_tma(1)
            assert_exact(y, ref, f"conv[{case[0]}] y on {label}", axes, tiles)
            results.append(y)
        assert all(torch.equal(results[0], r) for r in results[1:])


# ---- evk_conv2d_fwd -----------------------------------------------------------------------------------------------------
# B, H, W, C, N, k, stride, (dil_h, dil_w), act, (extra input channels, input channel offset), (output offset, extra):
# every wgmma column-tile boundary, M not a multiple of 128, stride 1 and 2
CONV2D_N_GRID = [(2, 13, 11, 24, n, 3, 2, (1, 1), a, (4, 0), (0, 3)) for n, a in ((32, 0), (33, 1), (64, 2), (65, 0), (128, 1), (129, 2))]
CONV2D_N_GRID += [(1, 19, 23, 40, n, 3, 1, (1, 1), a, (0, 0), (4, 0)) for n, a in ((32, 2), (33, 0), (65, 1), (129, 0))]
CONV2D_CASES = ([c[:7] + ((c[7], c[7]),) + c[8:] for c in CONV_GRID] + list(CONV_HW_GRID) + CONV2D_N_GRID)


def _conv2d_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.name for e in prof.events())


@pytest.mark.parametrize("case", CONV2D_CASES, ids=[f"c2d{i}" for i in range(len(CONV2D_CASES))])
def test_conv2d(ops, exact_mode, case):
    """wgmma (16-byte operands), mma.sync (the input slice shifted by one channel) and 3xTF32: all exact"""
    B, H, W, C, N, k, s, (dh, dw), act, (xe, xo), (yo, ye) = case
    L = exact_mode
    g = torch.Generator().manual_seed(B * 31 + H * 7 + C * 3 + N)
    x, w = R.ints((B, C, H, W), R.RX, g), R.ints((N, C, k, k), R.RW, g)
    scale, bias = R.ints((N,), 3, g, lo=1), R.ints((N,), R.RB, g)
    assert_bound(C * k * k * R.RX * R.RW, "conv2d")
    pad = (dh * (k // 2), dw * (k // 2))
    with torch.backends.cudnn.flags(enabled=False):
        pre = torch.nn.functional.conv2d(x.to(DEV), w.to(DEV), None, s, pad, (dh, dw))
    pre = (pre * scale.to(DEV)[:, None, None] + bias.to(DEV)[:, None, None]).permute(0, 2, 3, 1)
    p32 = pre.float()
    if act == 1:
        ref = torch.relu(pre)
    elif act == 2:                                       # one fp32 multiply by the fixed 0.01 slope
        ref = torch.where(p32 >= 0, p32, p32 * torch.tensor(0.01, dtype=torch.float32, device=DEV)).double()
    else:
        ref = pre
    Ho, Wo = ops.conv2d_out(H, k, s, pad[0], dh), ops.conv2d_out(W, k, s, pad[1], dw)
    wd = w.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    vec_ok = C % 4 == 0 and (C + xe) % 4 == 0 and xo % 4 == 0
    for label, shift, precise in (("as given", 0, False), ("shifted slice", 1, False), ("3xTF32", 0, True)):
        xbuf = torch.full((B, H, W, C + xe + shift), NAN, device=DEV)         # pitch padding and slack: NaN
        xbuf[..., xo + shift:xo + shift + C] = x.permute(0, 2, 3, 1).to(DEV)
        ybuf = torch.full((B, Ho, Wo, yo + N + ye), 7.0, device=DEV)
        L.evk_set_precise(1 if precise else 0)
        try:
            names = _conv2d_kernels(lambda: ops.conv2d(ops.CLView(xbuf, xo + shift, C), wd, ops.CLView(ybuf, yo, N), k=k, stride=s,
                                                       pad=pad, dil=(dh, dw), scale=scale.float().to(DEV), bias=bias.float().to(DEV),
                                                       act=act))
        finally:
            L.evk_set_precise(0)
        wgmma = "conv2d_fwd_wgmma" in names
        assert wgmma == (vec_ok and shift == 0 and not precise), (label, names)
        got = ybuf[..., yo:yo + N]
        if act == 3:
            err = float((got.double() - torch.sigmoid(pre)).abs().max())
            assert err <= 2e-6, (label, err)
        else:
            assert_exact(got, ref, f"conv2d {case} {label}", ("b", "ho", "wo", "n"), {"n": _bn(N)})
        assert (ybuf[..., :yo] == 7).all() and (ybuf[..., yo + N:] == 7).all(), label


# ---- the compensation contract at the default trunc_comp --------------------------------------------------------------
def _assert_compensated(got, exact, raw, tol_ulp, what):
    """outputs with |exact| >= 2^12 are within tol_ulp of exact * (1 + c)^raw and far from exact and exact * (1 + c)^(2 raw)"""
    c = torch.tensor(1.0, dtype=torch.float32) + torch.tensor(TRUNC_COMP, dtype=torch.float32)
    comp = float(c) ** raw
    got, exact = got.detach().double().flatten().to(DEV), exact.detach().double().flatten().to(DEV)
    sel = exact.abs() >= 2 ** 12
    assert int(sel.sum()) >= 1000, f"{what}: too few large outputs ({int(sel.sum())})"
    got, exact = got[sel], exact[sel]
    want = (exact * comp).float()
    ulp = (torch.nextafter(want.abs(), torch.tensor(math.inf, device=DEV)) - want.abs()).double()
    d = (got - want.double()).abs() / ulp
    assert float(d.max()) <= tol_ulp, f"{what}: {float(d.max()):.1f} ulp from exact * comp^{raw}"
    for other, label in ((exact, "uncompensated"), (exact * comp * comp, "compensated twice")):
        assert bool(((got - other).abs() / ulp > tol_ulp).all()), f"{what}: indistinguishable from the {label} result"


def test_compensation_applied_once(ops, exact_mode):
    L = exact_mode
    L.evk_set_tma_options(1, 1, TRUNC_COMP)
    g = torch.Generator().manual_seed(99)
    # raw operands = 1: Linear (flat path) and a tap-sum conv forward
    x, w = R.ints((1, 512, 2048), 3, g, lo=1), R.ints((64, 2048), 3, g, lo=1)
    with torch.no_grad():
        ops.dispatch_reset()
        y = ops.linear(x.float().to(DEV), ops.pack_weight(w.float().to(DEV).unsqueeze(-1)))
        torch.cuda.synchronize()
    assert_family(ops, "fwd_gemm_tma", FWD, "linear")
    _assert_compensated(y, x.to(DEV) @ w.to(DEV).t(), 1, 4, "linear")
    x, v = R.ints((2, 512, 600, 1), 3, g, lo=2), R.ints((64, 512, 3), 3, g, lo=2)
    with torch.no_grad():
        ops.dispatch_reset()
        y = ops.conv(_to_cl(x).float().to(DEV), ops.pack_weight(v.float().to(DEV)), pad=1)
        torch.cuda.synchronize()
    assert_family(ops, "fwd_gemm_tma", FWD, "tap-sum conv")
    _assert_compensated(y, _to_cl(R.conv1d_ref(x.to(DEV), v.to(DEV), None, 1, 1, 1)), 1, 4, "tap-sum conv")
    # raw operands = 2: evk_gemm_tf32 with one and with three K splits (each split's partial is scaled and rounded once)
    a, b = R.ints((300, 1024), 3, g, lo=2), R.ints((64, 1024), 3, g, lo=2)
    for splits in (1, 3):
        out = torch.zeros(300, 64, device=DEV)
        ops.dispatch_reset()
        ops.gemm_tf32(a.float().to(DEV), b.float().to(DEV), out=out, splits=splits)
        torch.cuda.synchronize()
        assert_family(ops, "gemm_tf32", FWD + WGRAD + ("gemm_tf32",), "gemm_tf32")
        _assert_compensated(out, a.to(DEV) @ b.to(DEV).t(), 2, 4 + splits, f"gemm_tf32 splits {splits}")
    # raw operands = 2: conv_wgrad_kernel, at a shape that runs one K split and at one that runs several
    for B, T, C, N, Q in ((1, 2048, 512, 512, 5), (2, 2048, 64, 64, 3)):
        x, v, gy = R.ints((B, C, T, 1), 3, g, lo=1), R.ints((N, C, Q), 1, g, lo=1), R.ints((B, N, T, 1), 3, g, lo=1)
        vd = v.float().to(DEV).requires_grad_(True)
        y = ops.conv(_to_cl(x).float().to(DEV), ops.pack_weight(vd), pad=Q // 2)
        ops.dispatch_reset()
        y.backward(_to_cl(gy).float().to(DEV))
        torch.cuda.synchronize()
        assert_family(ops, "wgrad_gemm_tma", WGRAD, "conv wgrad")
        tiles = Q * ((N + 127) // 128) * ((C + 127) // 128)                  # the split count evk_gconv_wgrad picks
        splits = max(1, min(64, torch.cuda.get_device_properties(DEV).multi_processor_count // tiles, B * ((T + 31) // 32) // 8))
        vr = v.to(DEV).requires_grad_(True)
        R.conv1d_ref(x.to(DEV), vr, None, 1, Q // 2, 1).backward(gy.to(DEV))
        _assert_compensated(vd.grad, vr.grad, 2, 4 + splits, f"conv wgrad B{B} C{C} N{N} splits {splits}")


def test_compensation_not_applied(ops, exact_mode):
    """gconv_tc, mma.sync and conv2d round their operands to nearest: no compensation, exact results at the default"""
    L = exact_mode
    L.evk_set_tma_options(1, 1, TRUNC_COMP)
    case = [c for c in R.CONV_CASES if c[0] == "tc npos 40 k3"][0]
    for label, fam, setup in (("gconv_tc", "fwd_gconv_tc", lambda: None), ("mma.sync", "fwd_mma_sync", lambda: L.evk_set_backend(0))):
        setup()
        try:
            with torch.no_grad():
                (_, y, ref, axes, tiles), = _run_conv(ops, case[:14] + (fam,) + case[15:], seed=23, backward=False, comp=TRUNC_COMP)
        finally:
            L.evk_set_backend(1)
        assert_exact(y, ref, f"{label} at the default compensation", axes, tiles)
    g = torch.Generator().manual_seed(4)
    x, w = R.ints((1, 64, 21, 32), R.RX, g), R.ints((64, 64, 3, 3), R.RW, g)
    y = torch.empty(1, 21, 32, 64, device=DEV)
    ops.conv2d(ops.CLView(x.permute(0, 2, 3, 1).float().contiguous().to(DEV)), w.float().permute(0, 2, 3, 1).contiguous().to(DEV),
               ops.CLView(y), k=3, pad=1)
    with torch.backends.cudnn.flags(enabled=False):
        ref = torch.nn.functional.conv2d(x.to(DEV), w.to(DEV), None, 1, 1).permute(0, 2, 3, 1)
    assert_exact(y, ref, "conv2d at the default compensation", ("b", "h", "w", "n"), None)
