"""Conv weight gradients on conv_wgrad_kernel (evk_gconv_wgrad given dY transposed), element for element against float64.

The kernel stacks (tap, input channel) pairs in its tile rows and reads X channels-last with the tap shift as a copy-engine
row coordinate.  With small-integer operands every product and partial sum is exact in fp32 (tests/exact_ref.py), so with
the truncation compensation off every dW element must equal the float64 result: a tap stacked into the wrong rows, a shift
off by one position, a dropped K block or split, or a transposed store into the wrong (n, c) changes an element by a
whole unit.  Every case asserts from the dispatch accounting that the weight-gradient flops ran on this kernel family.
"""
import pytest
import torch

from tests import exact_ref as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
TRUNC_COMP = 3.52e-4
WGRAD = ("wgrad_gemm_tma", "wgrad_mma_sync", "wgrad_direct")

# (label, B, T, C, N, k, stride, dil, P); pad = dil * (k - 1) // 2
CASES = [(f"k{k} d{d} 64ch", 2, 1100, 64, 64, k, 1, d, 1) for k in (3, 7, 11) for d in (1, 3, 5)]
CASES += [(f"k3 {c}ch", 2, 1100, c, c, 3, 1, 1, 1) for c in (32, 64, 128, 256)]
CASES += [
    ("k11 d5 32ch: three tap groups", 2, 2100, 32, 32, 11, 1, 5, 1),
    ("k5 C36 N96: taps straddle tiles", 2, 1100, 36, 96, 5, 1, 1, 1),
    ("C192 N384 k5", 2, 1100, 192, 384, 5, 1, 1, 1),
    ("P=3 k5 64ch", 2, 400, 64, 64, 5, 1, 1, 3),
    ("P=11 k5 128->64", 2, 100, 128, 64, 5, 1, 1, 11),
    ("stride 3 P=2 k5 phased", 4, 1000, 32, 128, 5, 3, 1, 2),
    ("stride 3 P=5 k5 phased", 3, 1200, 64, 64, 5, 3, 1, 5),
]


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    L = lib.init()
    L.evk_set_precise(0)
    L.evk_set_tma_options(1, 1, 0.0)
    try:
        yield ops
    finally:
        L.evk_set_tma_options(1, 1, TRUNC_COMP)


def _to_cl(t):
    B, C, T, P = t.shape
    return t.permute(0, 2, 3, 1).reshape(B, T * P, C)


def _splits(B, J, P, C, N, stride, Q):
    """the split count evk_gconv_wgrad picks for the largest stride phase"""
    nq = (Q + stride - 1) // stride
    tiles = nq * ((N + 127) // 128) * ((C + 127) // 128)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    return max(1, min(64, sms // tiles, B * ((J * P + 31) // 32) // 8))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_wgrad_exact(ops, case):
    _, B, T, C, N, k, stride, dil, P = case
    pad = dil * (k - 1) // 2
    J = R.conv_out_len(T, k, stride, pad, dil)
    g = torch.Generator().manual_seed(B * 1000 + T + C * 7 + N * 13 + k * 17 + dil + P * 31 + stride)
    x, v, gy = R.ints((B, C, T, P), R.RX, g), R.ints((N, C, k), R.RW, g), R.ints((B, N, J, P), R.RDY, g)
    assert B * J * P * R.RX * R.RDY <= R.EXACT_BOUND
    vd = v.float().to(DEV).requires_grad_(True)
    y = ops.conv(_to_cl(x).float().to(DEV), ops.pack_weight(vd), stride=stride, pad=pad, dil=dil, P=P)
    ops.dispatch_reset()
    y.backward(_to_cl(gy).float().to(DEV))
    torch.cuda.synchronize()
    st = ops.dispatch_stats()
    assert st["wgrad_gemm_tma"] > 0 and not any(st[f] for f in WGRAD[1:]), st
    vr = v.double().to(DEV).requires_grad_(True)
    R.conv1d_ref(x.double().to(DEV), vr, None, stride, pad, dil).backward(gy.double().to(DEV))
    got, want = vd.grad.double(), vr.grad
    bad = got != want
    if bool(bad.any()):
        idx = bad.nonzero()[:6].tolist()
        lines = [f"  [n={n}, c={c}, q={q}] got {float(got[n, c, q])!r} want {float(want[n, c, q])!r}" for n, c, q in idx]
        pytest.fail(f"{int(bad.sum())} of {bad.numel()} dW elements differ (splits {_splits(B, J, P, C, N, stride, k)})\n"
                    + "\n".join(lines))


def test_conv_wgrad_splits_reproducible(ops):
    """a shape that runs many K splits: two runs give the same bits"""
    B, T, C, N, k = 2, 2048, 64, 64, 7
    assert _splits(B, T, 1, C, N, 1, k) > 1
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, T, C, generator=g).to(DEV)
    v = torch.randn(N, C, k, generator=g).to(DEV)
    gy = torch.randn(B, T, N, generator=g).to(DEV)
    grads = []
    for _ in range(2):
        vd = v.clone().requires_grad_(True)
        ops.conv(x, ops.pack_weight(vd), pad=k // 2).backward(gy)
        grads.append(vd.grad.clone())
    assert torch.equal(grads[0], grads[1])


def _below_tf32(m, g):
    """integers m plus 0.5 .. 0.97 of a TF32 unit in the last place of |m|: the tensor core reads m itself (it truncates the
    low 13 mantissa bits), rounding to nearest would read m + ulp wherever the fraction is past one half"""
    ulp = torch.where(m.abs() >= 2, 2.0 ** -9, 2.0 ** -10).double()
    f = 0.5 + 0.47 * torch.rand(m.shape, generator=g, dtype=torch.float64)
    return (m.double() + torch.sign(m.double()) * f * ulp).float()


TRUNC_CASES = [c for c in CASES if c[0] in ("k3 32ch", "k7 d3 64ch", "k3 128ch", "k5 C36 N96: taps straddle tiles",
                                             "stride 3 P=2 k5 phased")]


@pytest.mark.parametrize("case", TRUNC_CASES, ids=[c[0] for c in TRUNC_CASES])
def test_conv_wgrad_truncates_both_operands(ops, case):
    """X and dY carry mantissa bits below TF32: dW must equal the exact result of their truncated (integer) values, the
    rounding the accumulator compensation of the library is calibrated for, whichever path each operand takes"""
    _, B, T, C, N, k, stride, dil, P = case
    pad = dil * (k - 1) // 2
    J = R.conv_out_len(T, k, stride, pad, dil)
    g = torch.Generator().manual_seed(T + C + N + k)
    x, v, gy = R.ints((B, C, T, P), R.RX, g), R.ints((N, C, k), R.RW, g), R.ints((B, N, J, P), R.RDY, g)
    vd = v.float().to(DEV).requires_grad_(True)
    y = ops.conv(_to_cl(_below_tf32(x, g)).to(DEV), ops.pack_weight(vd), stride=stride, pad=pad, dil=dil, P=P)
    ops.dispatch_reset()
    y.backward(_to_cl(_below_tf32(gy, g)).to(DEV))
    torch.cuda.synchronize()
    st = ops.dispatch_stats()
    assert st["wgrad_gemm_tma"] > 0 and not any(st[f] for f in WGRAD[1:]), st
    vr = v.double().to(DEV).requires_grad_(True)
    R.conv1d_ref(x.double().to(DEV), vr, None, stride, pad, dil).backward(gy.double().to(DEV))
    bad = vd.grad.double() != vr.grad
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} dW elements are not the result of truncated operands"
