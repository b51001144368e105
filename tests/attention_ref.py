"""Float64 references, per-element error bounds and a float32 emulator of the mma.sync attention kernels (csrc/attn_mma.cuh
under csrc/flash.cu and csrc/attn64.cu), for tests/test_gpu_attention_elementwise.py; tests/test_cpu_attention_ref.py
rehearses them on the CPU.

Error model.  Q, K, V and dO are small integers times a power of two (exact_ref.ints), so they are exact in TF32 whether the
tensor core truncates them (B operands enter as raw fp32 bits) or they were rounded to nearest (A operands, cvt.rna), and
every Q K^T and dO V^T is an exact fp32 integer.  What remains are these roundings, each named once below:
  - the fp32 products t = s * fp32(scale * log2e) and the fp32 differences t - m             U32 per operation
  - ex2.approx (SFU) for every probability and every online-rescale factor                      U_EX2, results < 2^-126 flush
                                                                                               to zero (TINY)
  - the TF32 rounding of the A operands P and dS of gemm_pn (split4)                           U_A (mode)
  - fp32 row sums, the fp32 dot product of delta, the fp32 multiplies by 1/l, 1/(1-p), scale   U32 per operation / term
  - the tensor core's fp32 accumulation: at most one truncation per added key                  U_ACC per key
  - with a non-exact rotary table only: the rotation and the truncation of the rotated K        U_B (mode)
Every bound below ("model") is the first-order propagation of these roundings, evaluated in float64 from absolute values.
The gate allows SAFETY = 2 times the model.  The factor is not fitted: one TF32 rounding of a probability alone can come
within a hair of its own first-order bound (2^-11 relative), so a gate equal to the model would leave nothing for what
the model leaves out -- second-order products of the roundings and the tensor core's unspecified accumulation order.
The CPU rehearsal checks that an fp32 emulation of the kernels stays within the model itself (half the gate) at every
element; the ratios the tests print are err / gate.  No constant comes
from a measurement.  Two kinds of output are exact by construction and required bit-exact: a masked probability
(ex2(-inf) = 0) and a dropped one (0.f).
"""
import math

import numpy as np
import torch

from oracle import gpt_oracle
from tests import exact_ref

LN2 = math.log(2.0)
LOG2E = 1.4426950408889634
U32 = 2.0 ** -24               # fp32 round-to-nearest, relative
U_EX2 = 2.0 ** -22             # ex2.approx.ftz.f32, relative
U_ACC = 2.0 ** -23             # one truncating fp32 addition in the tensor core, relative to the accumulated magnitude
TINY = 2.0 ** -126             # ex2.approx.ftz flushes smaller results to zero
SAFETY = 2.0                   # gate = SAFETY x first-order model
# U_A: relative error of an A operand (P, dS, rotated Q) as the tensor core sees it.  TF32: cvt.rna, 2^-11.  3xTF32: the
# residual of hi + lo, 2^-22.  U_B: a B operand fed as raw bits (the rotated K): truncation, 2^-10; 3xTF32: the lo part's
# rounding plus the dropped lo x lo product, 2^-21.
MODES = {"tf32": dict(UA=2.0 ** -11, UB=2.0 ** -10), "3xtf32": dict(UA=2.0 ** -22, UB=2.0 ** -21)}
FLASH_TILE, ATTN64_KEY_TILE = 64, 32     # keys per online-softmax step (flash.cu BT, attn64.cu BK)
PROB_FLOOR = 2.0 ** -40                  # visible probabilities of the mask-readout inputs stay at or above this


def fp32(x):
    return float(np.float32(x))


def sl2(scale):
    """the kernels' fp32 scale * log2e"""
    return fp32(np.float32(scale) * np.float32(LOG2E))


# ---- masks ------------------------------------------------------------------------------------------------------------
def flash_visible(xl, yl, X, L):
    """[B, L, L] bool, key j visible to query i: the prefix-LM mask of t2s_model.py (gpt_oracle.prefix_lm_mask)"""
    return ~gpt_oracle.prefix_lm_mask(torch.as_tensor(xl), torch.as_tensor(yl), X, L - X)


def flash_visible_kernel_rule(xl, yl, X, L):
    """the same mask written as flash.cu's allowed(i, j): used to move the prefix boundary in a modelled fault"""
    i, j = torch.arange(L)[:, None], torch.arange(L)[None, :]
    out = []
    for a, b in zip(torch.as_tensor(xl).tolist(), torch.as_tensor(yl).tolist()):
        out.append(torch.where(j < X, (j < a).expand(L, L), ((j - X) < b) & (j <= i)))
    return torch.stack(out)


def pad_visible(lens, L):
    """[B, L, L]: key j visible to every query row (padding rows included) iff j < clamp(lens, 1, L)"""
    n = torch.as_tensor(lens).clamp(1, L)
    return (torch.arange(L)[None, None, :] < n[:, None, None]).expand(len(n), L, L).clone()


def flash_key_tiles(i0, L, X, yl):
    """flash.cu key_tiles: the number of 64-key tiles a query tile starting at i0 streams"""
    jend = max(X, min(i0 + FLASH_TILE, L))
    jend = min(jend, X + yl)
    jend = max(jend, min(X, L))
    return (jend + FLASH_TILE - 1) // FLASH_TILE


# ---- dropout (flash.cu drop_key / drop_row / drop_col / drop_pair) ----------------------------------------------------
M32 = np.uint64(0xFFFFFFFF)
DROP_C, DROP_M1, DROP_M2 = 0xC2B2AE3D, 0x7FEB352D, 0x846CA68B


def _u32(x):
    return (np.asarray(x, dtype=np.uint64) & M32).astype(np.uint64)


def philox(seed, ctr, stream):
    """Philox-4x32-10 of evk_common.cuh: (c0, c1, c2, c3) for key = seed, counter = (ctr, stream)"""
    M = 0xFFFFFFFF
    c0, c1, c2, c3 = ctr & M, (ctr >> 32) & M, stream & M, (stream >> 32) & M
    a, b = seed & M, (seed >> 32) & M
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ a) & M, p1 & M, ((p0 >> 32) ^ c3 ^ b) & M, p0 & M
        a, b = (a + 0x9E3779B9) & M, (b + 0xBB67AE85) & M
    return c0, c1, c2, c3


def drop_threshold(p):
    """thr = round-down(p * 2^32) in double from the fp32 p, as drop_key computes it"""
    return int(min(max(float(np.float32(p)) * 4294967296.0, 1.0), 4294967295.0))


def drop_row(row, s0):
    x = _u32(np.asarray(row, dtype=np.uint64) * np.uint64(0x9E3779B1) + np.uint64(s0))
    x ^= x >> np.uint64(15); x = _u32(x * np.uint64(0x85EBCA77)); x ^= x >> np.uint64(13); x = _u32(x * np.uint64(0xC2B2AE35)); x ^= x >> np.uint64(16)
    return x


def drop_col(j, s1):
    return _u32((np.asarray(j, dtype=np.uint64) >> np.uint64(1)) * np.uint64(DROP_C) + np.uint64(s1))


def keep_matrix(z, L, s0, s1, p):
    """[L, L] keep flags of (batch * H + head) z: row hash of z * L + i (uint32), column pair term of j >> 1, M1 / M2 for
    even / odd j"""
    thr = np.uint64(drop_threshold(p))
    rh = drop_row(_u32(np.arange(L, dtype=np.uint64) + np.uint64(z * L)), s0)[:, None]
    cols = np.arange(L, dtype=np.uint64)
    h = rh ^ drop_col(cols, s1)[None, :]
    x = np.where((cols & np.uint64(1)).astype(bool)[None, :], _u32(h * np.uint64(DROP_M2)), _u32(h * np.uint64(DROP_M1)))
    return x >= thr


def keep_tensor(B, H, L, seed, offset, sid, p):
    """[B, H, L, L] keep flags of one flash launch with RNG state (seed, offset) and stream id sid"""
    s0, s1, _, _ = philox(int(seed), int(offset), int(sid))
    return torch.from_numpy(np.stack([keep_matrix(z, L, s0, s1, p) for z in range(B * H)])).view(B, H, L, L)


def drop_scale(keep, p):
    """keep / (1 - p) with the kernel's fp32 1 / (1 - p), as float64"""
    return keep.double() * fp32(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


# ---- float64 references ------------------------------------------------------------------------------------------------
def attention_ref(q, k, v, vis, scale, dscale=None):
    """q, k, v [..., L, d], vis [..., L, L] bool -> O, lse (log2 units), P (softmax, 0 where masked), t = s * scale * log2e.
    dscale (keep / (1 - p)) multiplies P before V.  Differentiable in q, k, v."""
    s = q @ k.transpose(-1, -2)
    logit = (s * scale).masked_fill(~vis, float("-inf"))
    P = torch.softmax(logit, -1)
    lse = torch.logsumexp(logit, -1) / LN2
    O = (P if dscale is None else P * dscale) @ v
    return O, lse, P, s * (scale * LOG2E)


def rope_rotate(x, cs):
    """interleaved rotation of x [..., L, 64] by cs [L, 32, 2] (cos, sin): out[2i] = x[2i] c - x[2i+1] s,
    out[2i+1] = x[2i+1] c + x[2i] s"""
    c, s = cs[..., 0].double().repeat_interleave(2, -1), cs[..., 1].double().repeat_interleave(2, -1)
    xp = x.unflatten(-1, (-1, 2))
    return x * c + torch.stack((-xp[..., 1], xp[..., 0]), -1).flatten(-2) * s


def rope_abs(x, cs):
    """|x[2i]| |c| + |x[2i+1]| |s| per rotated element: the magnitude its fp32 rounding is relative to"""
    c, s = cs[..., 0].double().abs().repeat_interleave(2, -1), cs[..., 1].double().abs().repeat_interleave(2, -1)
    xp = x.abs().unflatten(-1, (-1, 2))
    return x.abs() * c + torch.stack((xp[..., 1], xp[..., 0]), -1).flatten(-2) * s


# ---- bounds -------------------------------------------------------------------------------------------------------------
def fwd_model(t, vis, P, lse, absV, mode, tile, dscale=None, dt=None, out_extra=0.0):
    """First-order error model of O and lse of one online-softmax forward (flash_fwd_kernel, attn64_fwd_kernel).
    t: float64 logits in log2 units; dt: extra absolute error of t (a non-exact rotation); out_extra: extra relative
    error of the output scaling (the sigmoid gate).  -> (O bound [..., L, d], lse bound [..., L] in log2 units, E_t)"""
    UA = MODES[mode]["UA"]
    n = t.shape[-1]
    ntiles = -(-n // tile)
    tv = t.masked_fill(~vis, 0.0)
    m = tv.masked_fill(~vis, float("-inf")).amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    Et = U32 * (3 * tv.abs() + (tv - m).abs())
    if dt is not None:
        Et = Et + dt
    Et = Et * vis
    Emax = Et.amax(-1, keepdim=True)
    rescale = U_EX2 * (ntiles + 1) + 2 * U32 * ntiles           # ex2 of every p and rescale factor, the rescale multiplies
    eP = 2 * LN2 * Emax + rescale                                # relative error of a probability
    el = eP + n * U32                                            # of the row sum
    cO = eP + el + UA + U32 + n * U_ACC + 2 * U32 + out_extra    # + 1/(1-p), 1/l and its multiply
    D = vis.double() if dscale is None else dscale * vis
    if absV is None:                                             # V = identity: the readout of every probability
        bO = cO * (P * D) + TINY * D
    else:
        bO = cO * ((P * D) @ absV) + TINY * (D @ absV)
    Else = Emax[..., 0] + (rescale + n * U32) / LN2 + 3 * U32 * (lse.abs() + m[..., 0].abs())
    return bO, Else, Et


def flash_bwd_model(q, k, v, dO, vis, P, t, lse, O, bO, Else, Et, scale, mode, dscale=None):
    """First-order error model of dQ, dK, dV (flash_delta + flash_dq + flash_dkv).  The backward recomputes P from the
    forward's lse (error Else) and takes delta from the forward's O (error bO); dP = dO V^T is exact.  -> bounds of dQ, dK, dV
    (before the scale by `scale`, which is applied here)."""
    UA = MODES[mode]["UA"]
    n = t.shape[-1]
    D = vis.double() if dscale is None else dscale * vis
    g = (dO @ v.transpose(-1, -2)) * D
    gerr = 0.0 if dscale is None else U32 * g.abs()
    delta = (dO * O).sum(-1, keepdim=True)
    derr = (dO.abs() * bO).sum(-1, keepdim=True) + dO.shape[-1] * U32 * (dO.abs() * (O.abs() + bO)).sum(-1, keepdim=True)
    tv = t.masked_fill(~vis, 0.0)
    epb = (LN2 * (Et + Else[..., None] + U32 * (tv - lse[..., None]).abs()) + U_EX2) * vis
    dS = P * (g - delta)
    edS = dS.abs() * (epb + U32) + P * (gerr + derr + U32 * (g.abs() + delta.abs())) + TINY * (g - delta).abs() * vis
    A = edS + (UA + n * U_ACC) * dS.abs()
    PD = P * D
    fs = fp32(scale)
    bq = fs * (A @ k.abs()) + 2 * U32 * fs * (dS.abs() @ k.abs())
    bk = fs * (A.transpose(-1, -2) @ q.abs()) + 2 * U32 * fs * (dS.abs().transpose(-1, -2) @ q.abs())
    bv = ((PD * (epb + UA + U32 + n * U_ACC) + TINY * D).transpose(-1, -2)) @ dO.abs()
    return bq, bk, bv


# ---- float32 emulation of the kernel arithmetic -------------------------------------------------------------------------
def round_tf32(x):
    """cvt.rna.tf32.f32 of fp32 x by bit masking: round to 10 mantissa bits, ties away from zero"""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def a_operand(x, mode):
    """the value the tensor core multiplies for an fp32 A operand: tf32(x), or hi + lo (3xTF32, summed in float64)"""
    hi = round_tf32(x)
    if mode == "tf32":
        return hi.double()
    return hi.double() + round_tf32(x - hi).double()


def emulate_fwd(q, k, v, vis, scale, mode, keep=None, p=0.0):
    """fp32 emulation of one forward: exact scores, fp32 t and max, fp32 2^(t - m) (correctly rounded instead of
    ex2.approx, one pass instead of the online rescale), fp32 row sums, TF32 / 3xTF32 P, exact products accumulated in
    float64, fp32 1/l; v = None is the identity (the readout of every probability).  -> O, lse (float64 tensors holding
    fp32 values)"""
    s = (q @ k.transpose(-1, -2)).float()
    t = (s * torch.tensor(sl2(scale), dtype=torch.float32)).masked_fill(~vis, float("-inf"))
    m = t.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    pr = torch.exp2(t - m)
    pr = torch.where(pr < TINY, torch.zeros_like(pr), pr)
    l = pr.sum(-1, keepdim=True)
    if keep is not None:
        pr = torch.where(keep, pr * torch.tensor(fp32(1.0 / np.float32(1.0 - np.float32(p))), dtype=torch.float32), torch.zeros_like(pr))
    acc = (a_operand(pr, mode) if v is None else a_operand(pr, mode) @ v).float()
    O = acc * (1.0 / l)
    lse = m[..., 0] + torch.log2(l[..., 0])
    return O.double(), lse.double()


def emulate_bwd(q, k, v, dO, O, lse, vis, scale, mode, keep=None, p=0.0):
    """fp32 emulation of the backward from the forward's fp32 O and lse: fp32 delta, P = 2^(t - lse), fp32 dS,
    TF32 / 3xTF32 dS and P / (1 - p) as A operands.  -> dQ, dK, dV"""
    f = torch.float32
    delta = (dO.float() * O.float()).sum(-1, keepdim=True)
    t = (q @ k.transpose(-1, -2)).float() * torch.tensor(sl2(scale), dtype=f)
    pr = torch.where(vis, torch.exp2(t - lse.float()[..., None]), torch.zeros((), dtype=f))
    pr = torch.where(pr < TINY, torch.zeros_like(pr), pr)
    g = (dO @ v.transpose(-1, -2)).float()
    pd = pr
    if keep is not None:
        inv = torch.tensor(fp32(1.0 / np.float32(1.0 - np.float32(p))), dtype=f)
        g = torch.where(keep, g * inv, torch.zeros_like(g))
        pd = torch.where(keep, pr * inv, torch.zeros_like(pr))
    dS = pr * (g - delta)
    dSa = a_operand(dS, mode)
    fs = torch.tensor(fp32(scale), dtype=f)
    dQ = (dSa @ k).float() * fs
    dK = (dSa.transpose(-1, -2) @ q).float() * fs
    dV = (a_operand(pd, mode).transpose(-1, -2) @ dO).float()
    return dQ.double(), dK.double(), dV.double()


# ---- gates ---------------------------------------------------------------------------------------------------------------
def ratio(got, ref, model):
    """|got - ref| / (SAFETY * model) per element: inf where the model is 0 and got != ref, and inf where got is not
    finite (a NaN would otherwise compare as inside every gate)"""
    got = got.double().cpu()
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / (SAFETY * model))
    return torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))


def outside_gate(got, ref, model, zero=None):
    """bool per element: the error exceeds the gate, the output is not finite, or it is not exactly 0.0 where `zero` is set"""
    bad = ~(ratio(got, ref, model) <= 1)
    if zero is not None:
        bad |= zero & (got.double().cpu() != 0)
    return bad


def rel_l2(got, ref):
    got, ref = got.double().cpu(), ref.double()
    return float((got - ref).norm() / (ref.norm() + 1e-30))


def ints(shape, r, gen, lo=None):
    return exact_ref.ints(shape, r, gen, lo)


# ---- the GPU test's inputs ----------------------------------------------------------------------------------------------
FLASH_DK, ATTN64_DK = 32, 64
FLASH_READOUT_X = (0, 1, 63, 64, 65, 130)
FLASH_READOUT_Y = (1, 63, 64, 65, 200)
FLASH_SHIPPED = (256, 1024, (256, 200), (1024, 777))       # X, Y, xl, yl of the shipped training shape (B = 2)
PAD_READOUT_L = (1, 31, 32, 33, 63, 64, 65, 97, 130, 512)
PAD_LENS = (1, 31, 32, 33)                                  # + L, each clamped to L
DROP_P = (0.1, 0.25)
DROP_SHAPE = (3, 65, 130)                                   # B, X, Y of the dropout readout
DROP_SEED = 4242                                            # RNG state (DROP_SEED, 0) of every dropout launch
DROP_SID = 1                                                # and its stream id
ROPE_L = (1, 31, 32, 33, 62, 65, 801)
ROPE_H = 2
ROPE_REAL_L = 65
# general-V flash cases: name, B, H, X, Y, logit pattern, dropout p
FLASH_GENERAL = [("random", 3, 2, 70, 150, "random", 0.0), ("increasing", 2, 2, 64, 200, "increasing", 0.0),
                 ("decreasing", 2, 2, 65, 130, "decreasing", 0.0), ("spread", 2, 2, 33, 190, "spread", 0.0),
                 ("random-drop", 3, 2, 70, 150, "random", 0.1), ("increasing-drop", 2, 3, 63, 129, "increasing", 0.25)]


def flash_lens(X, Y):
    """every (xl, yl) of xl in {1, X/2, X} (xl = 0 without a prefix), yl in {1, Y-1, Y} (yl >= 1: a row with no visible
    key has no softmax)"""
    xs = sorted({1, max(X // 2, 1), X}) if X else [0]
    ys = sorted({1, max(Y - 1, 1), Y})
    pairs = [(a, b) for a in xs for b in ys]
    return torch.tensor([a for a, _ in pairs]), torch.tensor([b for _, b in pairs])


def readout_keys(L, H, block, r=0):
    """[H, block] key read by column c of head h when V of head h is the identity on key block (h + r) mod ceil(L / block);
    -1 past L"""
    nb = -(-L // block)
    j = (torch.arange(H)[:, None] + r) % nb * block + torch.arange(block)[None, :]
    return torch.where(j < L, j, torch.full_like(j, -1))


def readout_v(L, H, block, r=0):
    """[L, H * block] the probe V: V[j, h * block + c] = 1 iff j = readout_keys(...)[h, c]"""
    keys = readout_keys(L, H, block, r).reshape(-1)
    V = torch.zeros(L, H * block, dtype=torch.float64)
    ok = keys >= 0
    V[keys[ok], torch.arange(H * block)[ok]] = 1.0
    return V


def gather_readout(M, keys):
    """M [B, L, L] or [B, H, L, L] over keys -> [B, L, H, block] at the probe keys (0 where the key is past L)"""
    H, block = keys.shape
    if M.dim() == 3:
        M = M[:, None].expand(M.shape[0], H, *M.shape[1:])
    idx = keys.clamp(min=0)[None, :, None, :].expand(M.shape[0], H, M.shape[2], block)
    out = torch.gather(M, 3, idx) * (keys >= 0)[None, :, None, :]
    return out.permute(0, 2, 1, 3)


def readout_qk(B, L, dk, seed):
    """shared Q, K of the mask readout: entries in {-1, 0, 1}, so |t| <= dk * scale * log2e and a visible probability is at
    least 2^-(2 max |t| + log2 L)"""
    g = torch.Generator().manual_seed(seed)
    return ints((B, L, dk), 1, g), ints((B, L, dk), 1, g)


def readout_ref(q, k, vis, scale, mode, tile, dscale=None):
    """P (times dscale) for every (query, key) and its model bound: q, k [B, 1, L, d], vis [B, L, L], dscale [B, H, L, L]
    -> ref, model [B, 1 or H, L, L], and the undropped P [B, 1, L, L]"""
    v4 = vis[:, None]
    _, lse, P, t = attention_ref(q, k, q[..., :1], v4, scale)
    model, _, _ = fwd_model(t, v4, P, lse, None, mode, tile, dscale=dscale)
    return (P if dscale is None else P * dscale), model, P


def flash_general_inputs(B, H, X, Y, pattern, seed):
    """q, k, v, dO [B, H, L, 32] and xl, yl of a general-V case.  'increasing' / 'decreasing' add a key ramp to one
    column so the row maximum rises (every tile rescales) or stays on the first tile; 'spread' makes logits span
    hundreds of log2 units so that most probabilities underflow."""
    g = torch.Generator().manual_seed(seed)
    L = X + Y
    q, k, v, do = (ints((B, H, L, FLASH_DK), r, g) for r in (3, 3, 3, 2))
    j = torch.arange(L, dtype=torch.float64)
    if pattern in ("increasing", "decreasing"):
        q[..., 0] = 4.0
        k[..., 0] = (j // 8) if pattern == "increasing" else -(j // 8)
    elif pattern == "spread":
        q[..., 0] = 16.0
        k[..., 0] = (j * 37) % 101 - 50
    xl = torch.randint(max(X // 2, 1), X + 1, (B,), generator=g); xl[0] = X
    yl = torch.randint(max(Y // 2, 1), Y + 1, (B,), generator=g); yl[0] = Y
    return q, k, v, do, xl, yl


def quarter_turn_cs(L):
    """[L, 32, 2] (cos, sin) of quarter turns whose number depends on the position and the pair: the rotation is exact"""
    p, i = torch.arange(L)[:, None], torch.arange(32)[None, :]
    n = (p + 3 * i + p * i) % 4
    c = torch.tensor([1.0, 0.0, -1.0, 0.0])[n]
    s = torch.tensor([0.0, 1.0, 0.0, -1.0])[n]
    return torch.stack([c, s], -1).float()


def rope_inputs(n, H, L, seed):
    """q, k, v [n, H, L, 64] and gate logits [n, H, L] (a distinct value per row and head)"""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (ints((n, H, L, ATTN64_DK), 2, g) for _ in range(3))
    gate = ((torch.arange(n)[:, None, None] * 5 + torch.arange(H)[None, :, None] * 3 + torch.arange(L)[None, None, :] * 7) % 23
            - 11).double() / 4.0
    return q, k, v, gate


GATE_U = 8 * U32        # expf, 1 + e, the product with l and the reciprocal of the gate scaling


def rope_ref(q, k, v, gate, cs, mode):
    """-> O (float64) and its model bound for evk_rope_attn_fwd: q, k rotated by cs, scale 1/8, times sigmoid(gate).
    A non-exact table adds the rotations' fp32 rounding and the A / B operand rounding of the rotated Q / K to t."""
    L = q.shape[-2]
    qr, kr = rope_rotate(q, cs[:L]), rope_rotate(k, cs[:L])
    vis = torch.ones(q.shape[:-2] + (L, L), dtype=torch.bool)
    O, lse, P, t = attention_ref(qr, kr, v, vis, 0.125)
    cs64 = cs[:L].double()
    exact = bool(((cs64 == 0) | (cs64.abs() == 1)).all())
    dt = None
    if not exact:
        m = MODES[mode]
        dt = sl2(0.125) * (m["UA"] + m["UB"] + 4 * U32) * (rope_abs(q, cs[:L]) @ rope_abs(k, cs[:L]).transpose(-1, -2))
    bO, _, _ = fwd_model(t, vis, P, lse, v.abs(), mode, ATTN64_KEY_TILE, dt=dt, out_extra=GATE_U)
    sg = torch.sigmoid(gate)[..., None]
    return O * sg, bO * sg
