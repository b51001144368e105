"""Float64 references and case tables of the exact-operand contraction tests (tests/test_gpu_exact_contractions.py; the
CPU half is rehearsed by tests/test_cpu_exact_contractions.py).

The operands of those tests are small integers.  An integer with at most 11 significant bits is exact in TF32, whether
the tensor core truncates it (raw TMA operands) or it was rounded to nearest (packed weights, cvt.rna), so every product
is an exact integer.  As long as sum_k |a_k| |b_k| <= 2^20 for every output, every partial sum is an exact fp32 integer
too: the tensor core's alignment to the largest exponent drops no bits and the order of the additions does not matter.
With the truncation compensation off, every kernel must then reproduce the float64 result bit for bit, and a wrong
index shows up as an error of at least one unit at the output it touched.
"""
import torch
import torch.nn.functional as F

EXACT_BOUND = 2 ** 20

# value ranges (inclusive, symmetric): activations, weights, upstream gradients, bias / residual
RX, RW, RDY, RB = 3, 2, 2, 4
LRELU_SLOPE = 0.25            # exact in binary: the leaky-ReLU derivative keeps gradients on a grid of 1/4
ACT_NONE, ACT_LRELU, ACT_RELU, ACT_TANH, ACT_GELU = 0, 1, 2, 3, 4


def ints(shape, r, gen, lo=None):
    """uniform integers in [lo, r] (lo = -r by default) as float64 on the CPU"""
    lo = -r if lo is None else lo
    return torch.randint(lo, r + 1, tuple(shape), generator=gen, dtype=torch.int64).double()


def conv_out_len(T, Q, stride, pad, dil):
    return (T + 2 * pad - dil * (Q - 1) - 1) // stride + 1


def conv1d_ref(x, w, bias=None, stride=1, pad=0, dil=1, groups=1):
    """Conv1d over a period-folded input by unfold + matmul: x [B, C, T, P], w [N, C / groups, Q] -> [B, N, J, P]
    (P = 1 is the plain Conv1d; P > 1 is Conv2d with a (Q, 1) kernel over [B, C, T, P])."""
    B, C, T, P = x.shape
    N, Cg, Q = w.shape
    J = conv_out_len(T, Q, stride, pad, dil)
    xp = F.pad(x, (0, 0, pad, pad))
    idx = (torch.arange(J)[:, None] * stride + torch.arange(Q)[None, :] * dil).to(x.device)     # [J, Q]
    cols = xp[:, :, idx, :].reshape(B, groups, Cg, J, Q, P)
    y = torch.einsum("bgcjqp,gncq->bgnjp", cols, w.reshape(groups, N // groups, Cg, Q)).reshape(B, N, J, P)
    return y if bias is None else y + bias.reshape(1, N, 1, 1)


def conv_transpose1d_ref(x, v, bias=None, stride=1, pad=0):
    """ConvTranspose1d by scattering each tap's matmul: x [B, Cin, T], v [Cin, Cout, Q] -> [B, Cout, (T-1) s - 2 pad + Q]"""
    B, Cin, T = x.shape
    Q = v.shape[2]
    full = (T - 1) * stride + Q
    parts = []
    for q in range(Q):
        yq = torch.einsum("bct,cd->bdt", x, v[:, :, q])                      # lands on positions t * stride + q
        parts.append(F.pad(yq.unsqueeze(-1), (0, stride - 1)).flatten(2)[:, :, :(T - 1) * stride + 1])
    y = sum(F.pad(p, (q, full - q - p.shape[2])) for q, p in enumerate(parts))
    y = y[:, :, pad:full - pad]
    return y if bias is None else y + bias.reshape(1, -1, 1)


def act_ref(t, act, slope=LRELU_SLOPE):
    if act == ACT_LRELU:
        return F.leaky_relu(t, slope)
    if act == ACT_RELU:
        return torch.relu(t)
    if act == ACT_TANH:
        return torch.tanh(t)
    return t


# ---- case tables ------------------------------------------------------------------------------------------------------
# evk_gemm_tf32: M, N, K, epilogue ("none", "brr" = bias + residual + ReLU, "lrelu" = bias + LReLU(0.25))
# M crosses 1 / 128 / 256-row tiles and has more 128-row tiles than the 132 SMs; N = 4 / 33 / 65 / 129 / 130 covers the
# 32 / 64 / 128-column tiles and the slow epilogue (N % 4 != 0); K = 4 / 31 / 33 / 200 covers the 32-column K tails.
GEMM_CASES = [
    (1, 4, 4, "none"), (127, 33, 31, "brr"), (129, 65, 33, "lrelu"), (257, 129, 200, "brr"), (132 * 128 + 1, 130, 33, "brr"),
    (129, 130, 4, "lrelu"), (257, 4, 200, "none"), (127, 129, 33, "none"), (132 * 128 + 1, 33, 200, "lrelu"),
    (1, 130, 200, "brr"), (257, 64, 31, "brr"), (132 * 128 + 1, 128, 64, "lrelu"),
]
# split-K into an integer-initialised D, operands in {-1, 0, 1}: M, N, K, splits (64 > the K blocks of the last one)
SPLITK_CASES = [(512, 384, 8192, 8), (200, 130, 1000, 5), (129, 64, 4096, 2), (300, 64, 1000, 64)]
# Linear (1x1 conv) through evk_gconv_fwd on the flat GEMM path: B, T, C, N, epilogue (B > 1 folds into rows)
LINEAR_CASES = [(1, 512, 64, 64, "brr"), (3, 171, 68, 96, "lrelu"), (1, 4097, 512, 1536, "none"), (4, 1024, 512, 96, "brr"),
                (2, 2049, 68, 1536, "lrelu")]
# Linear launches of a few rows on both sides of each rule of evk_gconv_fwd's route 0 (evk_gemv_rows, exact fp32): name, B, T,
# C, N, act, residual, no_grad, dispatch slot.  The staging limit is pow2(rows) * C <= 10240 (rows 3 count as 4).
GEMV_CASES = [
    ("rows 4", 1, 4, 512, 96, ACT_RELU, False, True, "fwd_gemv"),
    ("rows 5", 1, 5, 512, 96, ACT_RELU, False, True, "fwd_gconv_tc"),
    ("rows 4 as batch", 4, 1, 512, 96, ACT_LRELU, False, True, "fwd_gemv"),
    ("rows 3 C 2560", 1, 3, 2560, 96, ACT_NONE, False, True, "fwd_gemv"),
    ("rows 3 C 2564", 1, 3, 2564, 96, ACT_NONE, False, True, "fwd_gconv_tc"),
    ("rows 1 C 10240", 1, 1, 10240, 64, ACT_NONE, False, True, "fwd_gemv"),
    ("rows 1 C 10244", 1, 1, 10244, 64, ACT_NONE, False, True, "fwd_gconv_tc"),
    ("C 64", 1, 2, 64, 96, ACT_NONE, False, True, "fwd_gemv"),
    ("C 66", 1, 2, 66, 96, ACT_NONE, False, True, "fwd_direct"),
    ("grad enabled", 1, 2, 512, 96, ACT_RELU, False, False, "fwd_gconv_tc"),
    ("res", 1, 2, 512, 96, ACT_RELU, True, True, "fwd_gconv_tc"),
    ("gelu", 1, 2, 512, 96, ACT_GELU, False, True, "fwd_gconv_tc"),
]

# Conv cases through ops.conv: name, B, Tin, C, N, Q, stride, pad, dil, P, groups, act, res, masks ("" / "out" / "inout"),
# forward family, data-gradient family (None: not asserted; "-": no backward, e.g. tanh), weight-gradient family,
# TMA options (slab, mt2) and optionally a mode: "x+1" (x starts one float into its rows: not 16-byte aligned) or
# "precise" (3xTF32 products, evk_set_precise).
CONV_CASES = [
    # the "TMA ..." shapes of tests/checks.py check_conv (the s3 p=2 one at Tin = 1000: at 341 it is below the phased
    # path's 2048-row threshold and runs on mma.sync)
    ("tma resblock k11 d1 128ch +res", 3, 1500, 128, 128, 11, 1, 5, 1, 1, 1, ACT_LRELU, True, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma resblock k7 d5 64ch", 2, 2100, 64, 64, 7, 1, 15, 5, 1, 1, ACT_LRELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma conv_pre k7 192->512", 5, 500, 192, 512, 7, 1, 3, 1, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma discP 512->1024 k5 s1 p=3", 3, 310, 512, 1024, 5, 1, 2, 1, 3, 1, ACT_LRELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma k3 36->96 C tail", 2, 1100, 36, 96, 3, 1, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma discP 128->512 k5 s3 p=2 phased", 4, 1000, 128, 512, 5, 3, 2, 1, 2, 1, ACT_LRELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma discP 32->128 k5 s3 p=5 phased", 3, 410, 32, 128, 5, 3, 2, 1, 5, 1, ACT_NONE, False, "", "fwd_gemm_tma", None, "wgrad_gemm_tma", (1, 1)),
    ("tma ssl_proj k2 s2 768 phased", 6, 700, 768, 768, 2, 2, 0, 1, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("tma k41 s4 64 phased", 3, 3000, 64, 64, 41, 4, 20, 1, 1, 1, ACT_LRELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    # slab spans 1 and 256, the same span-256 case without the slab, and span 300 (> 256: the per-tap ring)
    ("slab span 1 k2", 2, 1200, 64, 64, 2, 1, 0, 1, 1, 1, ACT_RELU, True, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("slab span 256 k3 d128", 2, 1100, 32, 96, 3, 1, 128, 128, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("no slab span 256 k3 d128", 2, 1100, 32, 96, 3, 1, 128, 128, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (0, 1)),
    ("ring span 300 k11 d30", 2, 1100, 64, 64, 11, 1, 150, 30, 1, 1, ACT_LRELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    # N = 32 over 2 x 16000 rows: the cost model picks 256-row tiles (mt2 on) -- and 128-row tiles with it off
    ("mt2 N=32 256-row tiles", 2, 16000, 32, 32, 3, 1, 1, 1, 1, 1, ACT_LRELU, True, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("mt2 off N=32", 2, 16000, 32, 32, 3, 1, 1, 1, 1, 1, ACT_LRELU, True, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 0)),
    # period folds, output-length masks, residuals
    ("P=2 k5 +out_len", 2, 600, 32, 64, 5, 1, 2, 1, 2, 1, ACT_RELU, False, "out", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("P=3 k3 +res", 2, 400, 64, 32, 3, 1, 1, 1, 3, 1, ACT_LRELU, True, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("P=5 k5 +out_len", 3, 140, 36, 64, 5, 1, 2, 1, 5, 1, ACT_NONE, False, "out", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("P=11 k5", 2, 100, 64, 128, 5, 1, 2, 1, 11, 1, ACT_LRELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    # in_len with a period fold: the forward reads rows t*P + w with t >= in_len as zero, so those rows of dx are zero
    ("P=2 k5 +in_len", 3, 40, 32, 32, 5, 1, 2, 1, 2, 1, ACT_NONE, False, "inout", "fwd_gconv_tc", None, "wgrad_mma_sync", (1, 1)),
    ("phased s2 P=2 k4", 2, 1100, 64, 64, 4, 2, 1, 1, 2, 1, ACT_RELU, False, "", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    ("phased s4 P=5 k8 +out_len", 2, 1000, 32, 64, 8, 4, 2, 1, 5, 1, ACT_NONE, False, "out", "fwd_gemm_tma", "fwd_gemm_tma", "wgrad_gemm_tma", (1, 1)),
    # gconv_tc_kernel: in_len-masked input (WN in_layer), 16-channel resblock, grouped (DiscriminatorS groups at stride 1),
    # npos < 64; then the strided grouped DiscriminatorS layers, whose data gradient runs on it
    ("tc wn in_layer k5 +in_len", 3, 70, 192, 384, 5, 1, 2, 1, 1, 1, ACT_NONE, False, "inout", "fwd_gconv_tc", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("tc resblock k7 d3 c16 +res", 2, 515, 16, 16, 7, 1, 9, 3, 1, 1, ACT_LRELU, True, "", "fwd_gconv_tc", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("tc grouped g4 16->64 k41", 2, 300, 16, 64, 41, 1, 20, 1, 1, 4, ACT_LRELU, False, "", "fwd_gconv_tc", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("tc grouped g64 256->1024 k41", 2, 130, 256, 1024, 41, 1, 20, 1, 1, 64, ACT_LRELU, False, "", "fwd_gconv_tc", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("tc npos 40 k3", 4, 40, 64, 64, 3, 1, 1, 1, 1, 1, ACT_RELU, False, "", "fwd_gconv_tc", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("tc P=3 npos 69 1024ch", 2, 23, 1024, 1024, 5, 1, 2, 1, 3, 1, ACT_LRELU, False, "", "fwd_gconv_tc", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("discS 16->64 k41 s4 g4", 2, 1000, 16, 64, 41, 4, 20, 1, 1, 4, ACT_LRELU, False, "", "fwd_mma_sync", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    ("discS 256->1024 k41 s4 g64", 2, 130, 256, 1024, 41, 4, 20, 1, 1, 64, ACT_LRELU, False, "", "fwd_mma_sync", "fwd_gconv_tc", "wgrad_mma_sync", (1, 1)),
    # mma.sync: strided below the phased threshold, ragged and grouped weight gradients
    ("mma discP 32->128 k5 s3 p=2", 2, 119, 32, 128, 5, 3, 2, 1, 2, 1, ACT_LRELU, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("tc wn k5 20->44 +in_len ragged", 2, 37, 20, 44, 5, 1, 2, 1, 1, 1, ACT_NONE, False, "inout", "fwd_gconv_tc", None, "wgrad_mma_sync", (1, 1)),
    # direct fp32 kernels: channel counts that are not multiples of 4
    ("direct C=6 k5", 2, 300, 6, 32, 5, 1, 2, 1, 1, 1, ACT_LRELU, False, "", "fwd_direct", None, "wgrad_direct", (1, 1)),
    ("direct C=2 k5 s3 P=5", 2, 200, 2, 32, 5, 3, 2, 1, 5, 1, ACT_LRELU, False, "", "fwd_direct", None, "wgrad_direct", (1, 1)),
    # the routing rules on both sides of each threshold: phase-split TMA forward and TMA weight gradient for strided convs
    # (B*J*P >= 2048, J*P >= 64, C >= 32, N >= 32, stride <= 4, 16-byte x, no in_len, not precise), grouped convs
    ("route B*J*P 2047 s2", 1, 4093, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("route B*J*P 2048 s2", 1, 4095, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", None, "wgrad_gemm_tma", (1, 1)),
    ("route J*P 63 s2", 33, 125, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("route J*P 64 s2", 32, 127, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_gemm_tma", None, "wgrad_gemm_tma", (1, 1)),
    ("route C 28 s2", 1, 4095, 28, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("route N 28 s2", 1, 4095, 32, 28, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("route stride 5", 3, 4000, 32, 32, 5, 5, 2, 1, 1, 1, ACT_NONE, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("route x+1 s2", 1, 4095, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_direct", None, "wgrad_direct", (1, 1, "x+1")),
    ("route in_len s2", 1, 4095, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "inout", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1)),
    ("route precise s2", 1, 4095, 32, 32, 3, 2, 1, 1, 1, 1, ACT_NONE, False, "", "fwd_mma_sync", None, "wgrad_mma_sync", (1, 1, "precise")),
    ("route grouped g2 8->6 Ng 3", 2, 300, 8, 6, 5, 1, 2, 1, 1, 2, ACT_NONE, False, "", "fwd_gconv_tc", None, "wgrad_direct", (1, 1)),
    # N / G = 3: the strided grouped data gradient takes the direct kernel, the forward mma.sync
    ("route grouped g2 8->6 Ng 3 s2", 2, 300, 8, 6, 5, 2, 2, 1, 1, 2, ACT_LRELU, False, "", "fwd_mma_sync", "fwd_direct", "wgrad_direct", (1, 1)),
    # group slices that are not 16-byte tileable (C / G = 3): the direct kernels take the grouped conv as G
    ("route grouped g2 6->8 Cg 3", 2, 300, 6, 8, 5, 1, 2, 1, 1, 2, ACT_LRELU, False, "", "fwd_direct", "fwd_direct", "wgrad_direct", (1, 1)),
]
# conv_post: 16 -> 1 channel carried as 4 (zero weight rows), tanh: B, Tin, C, Q, pad
CONV_POST = (2, 700, 16, 7, 3)
# ConvTranspose1d, the shapes of check_conv_transpose that run on the TMA kernel: Cin, Cout, Q, stride, T, and optionally
# "x+1" (x starts one float into its rows: not 16-byte aligned, so the forward and the weight gradient run on the direct kernels)
CONVT_CASES = [(256, 128, 16, 8, 1100), (64, 32, 4, 2, 1500), (128, 64, 8, 2, 130), (64, 32, 4, 2, 300, "x+1")]


def conv_case_bounds(case):
    """-> the largest sum_k |a_k| |b_k| any output of the case's forward, data gradient and weight gradient can reach, from
    the shapes and value ranges alone (gradients through LReLU(0.25) are counted in units of 1/4)."""
    name, B, Tin, C, N, Q, stride, pad, dil, P, G, act, res, masks = case[:14]
    J = conv_out_len(Tin, Q, stride, pad, dil)
    unit = 4 if act == ACT_LRELU else 1
    fwd = (C // G) * Q * RX * RW
    dgrad = (N // G) * Q * RDY * RW * unit
    wgrad = B * J * P * RX * RDY * unit
    return fwd, dgrad, wgrad


def gemm_case_bound(K, ra=RX, rb=RW):
    return K * ra * rb
