"""CPU rehearsal of the exact-operand contraction tests (tests/test_gpu_exact_contractions.py): the float64 reference
helpers agree with torch's convolutions, and every case in the tables keeps its sums exact in fp32."""
import pytest
import torch
import torch.nn.functional as F

from tests import exact_ref as R


@pytest.mark.parametrize("B,C,N,T,P,Q,stride,pad,dil,groups", [
    (2, 6, 8, 37, 1, 5, 1, 2, 1, 1), (2, 8, 12, 40, 1, 3, 1, 4, 4, 1), (3, 4, 8, 29, 3, 5, 3, 2, 1, 1),
    (2, 8, 16, 50, 1, 7, 4, 3, 1, 4), (1, 8, 8, 33, 5, 2, 2, 0, 1, 2), (2, 5, 3, 11, 2, 4, 1, 1, 2, 1),
])
def test_conv1d_ref_matches_torch(B, C, N, T, P, Q, stride, pad, dil, groups):
    g = torch.Generator().manual_seed(B + C + N + T)
    x = R.ints((B, C, T, P), R.RX, g).requires_grad_(True)
    w = R.ints((N, C // groups, Q), R.RW, g).requires_grad_(True)
    b = R.ints((N,), R.RB, g).requires_grad_(True)
    y = R.conv1d_ref(x, w, b, stride, pad, dil, groups)
    xt, wt, bt = [t.detach().clone().requires_grad_(True) for t in (x, w, b)]
    yt = F.conv2d(xt, wt.unsqueeze(-1), bt, (stride, 1), (pad, 0), (dil, 1), groups)
    assert torch.equal(y, yt)
    gy = R.ints(y.shape, R.RDY, g)
    y.backward(gy)
    yt.backward(gy)
    for a, t in ((x, xt), (w, wt), (b, bt)):                 # data gradient (strided: the polyphase scatter), dW, dbias
        assert torch.equal(a.grad, t.grad)


@pytest.mark.parametrize("Cin,Cout,Q,stride,T", [(6, 4, 16, 8, 9), (4, 3, 4, 2, 15), (5, 2, 8, 2, 7), (3, 4, 3, 1, 10), (2, 2, 2, 2, 5)])
def test_conv_transpose1d_ref_matches_torch(Cin, Cout, Q, stride, T):
    g = torch.Generator().manual_seed(Cin * Q + T)
    pad = (Q - stride) // 2
    x = R.ints((2, Cin, T), R.RX, g).requires_grad_(True)
    v = R.ints((Cin, Cout, Q), R.RW, g).requires_grad_(True)
    b = R.ints((Cout,), R.RB, g)
    y = R.conv_transpose1d_ref(x, v, b, stride, pad)
    xt, vt = x.detach().clone().requires_grad_(True), v.detach().clone().requires_grad_(True)
    yt = F.conv_transpose1d(xt, vt, b, stride=stride, padding=pad)
    assert torch.equal(y, yt)
    gy = R.ints(y.shape, R.RDY, g)
    y.backward(gy)
    yt.backward(gy)
    assert torch.equal(x.grad, xt.grad) and torch.equal(v.grad, vt.grad)


def test_case_tables_stay_exact():
    """sum |a||b| <= 2^20 for every output of every case, from the shapes and value ranges alone"""
    for M, N, K, epi in R.GEMM_CASES:
        assert R.gemm_case_bound(K) <= R.EXACT_BOUND, (M, N, K)
    for M, N, K, splits in R.SPLITK_CASES:
        assert R.gemm_case_bound(K, 1, 1) + 100 <= R.EXACT_BOUND, (M, N, K)
    for B, T, C, N, epi in R.LINEAR_CASES:
        assert R.gemm_case_bound(C) <= R.EXACT_BOUND, (B, T, C, N)
    for case in R.CONV_CASES:
        for what, bound in zip(("forward", "data gradient", "weight gradient"), R.conv_case_bounds(case)):
            assert bound <= R.EXACT_BOUND, (case[0], what, bound)
    B, T, C, Q, pad = R.CONV_POST
    assert C * Q * R.RX * R.RW <= R.EXACT_BOUND
    for Cin, Cout, Q, s, T in (c[:5] for c in R.CONVT_CASES):
        assert Cin * -(-Q // s) * R.RX * R.RW <= R.EXACT_BOUND
        assert Cout * Q * R.RDY * R.RW <= R.EXACT_BOUND and 2 * T * R.RX * R.RDY <= R.EXACT_BOUND


def test_case_tables_reach_their_paths():
    """shape-level preconditions of the dispatch each case names (the GPU test checks the dispatch itself)"""
    for name, B, Tin, C, N, Q, stride, pad, dil, P, G, act, res, masks, ffam, dfam, wfam, opts in R.CONV_CASES:
        J = R.conv_out_len(Tin, Q, stride, pad, dil)
        assert J > 0, name
        if wfam == "wgrad_gemm_tma":                 # the library's TMA weight-gradient eligibility
            assert B * J * P >= 2048 and J * P >= 64 and C >= 32 and N >= 32 and C % 4 == 0 and G == 1 and not masks.startswith("in"), name
        if ffam == "fwd_gemm_tma" and stride > 1:    # the phased strided forward
            assert B * J * P >= 2048 and J * P >= 64 and C % 4 == 0 and C >= 32 and N >= 32, name
    spans = {c[0]: (c[5] - 1) * c[8] * c[9] for c in R.CONV_CASES if c[6] == 1 and c[5] > 1 and c[14] == "fwd_gemm_tma"}
    assert min(spans.values()) == 1 and 256 in spans.values() and max(spans.values()) > 256
