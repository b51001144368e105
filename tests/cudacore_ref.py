"""Float64 references and per-element error bounds for the fp32 CUDA-core training kernels (csrc/norm_weights.cu,
csrc/elementwise.cu, csrc/gpt_misc.cu, csrc/vq_loss_optim.cu and the fixed-order cross-block sum ordered_sum of
csrc/api.cu), for tests/test_gpu_cudacore_elementwise.py; tests/test_cpu_cudacore_ref.py rehearses them on the CPU against
fp32 emulations of the kernels' summation orders.

Error model.  The library is built without --use_fast_math, so every fp32 +, -, *, / and sqrtf rounds correctly
(U32 = 2^-24 relative per operation; an FMA the compiler contracts rounds once, which the model over-covers).  The
transcendentals carry the CUDA Programming Guide's maximum ulp errors (ULPS below); one ulp of a normal result r is at
most 2^-23 |r|.  __expf(x) (sigmoidf_, reparam, the KL loss) is ex2.approx(x log2 e) with 2 + floor(|1.173 x|) ulp, a term
that grows with the argument.  A value is carried as E(v, e): v the float64 value of the operation on the fp32 inputs,
e a first-order bound of |fp32 result - v| that every operation propagates (|df/da| e_a + ...) and to which it adds its
own rounding.  A sum of n terms adds (its longest addition chain) * U32 * sum |term|; the chain of each kernel is taken
from its order -- lane-strided partial sums, the warp_sum / block_sum butterflies, per-block partials, ordered_sum's
16 lanes -- and written next to the kernel below.  The gate is SAFETY * model; SAFETY = 2 leaves room for what a
first-order model leaves out.  No constant is fitted to a GPU measurement.  Outputs that are exact by construction
(masked and padded zeros, copies, gathers, transposes, counts) have e = 0 and must be bit-exact.
"""
import math

import torch

U32 = 2.0 ** -24                 # fp32 round to nearest, relative
ULP = 2.0 ** -23                 # one ulp of a normal fp32 result, relative
TINY = 2.0 ** -149               # one ulp of the smallest subnormal: the floor of any result's rounding
SAFETY = 2.0
ULPS = dict(exp=2, tanh=2, log=1, log1p=1, erf=2, rsqrt=2)
NUM_SMS = 132
OS_LANES = 16                    # ordered_sum: lanes per output column
F64 = torch.float64


def cdiv(a, b):
    return -(-a // b)


class E:
    """float64 value and first-order absolute error bound of an fp32 computation"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = torch.as_tensor(v, dtype=F64)
        self.e = torch.zeros_like(self.v) if e is None else torch.as_tensor(e, dtype=F64) * torch.ones_like(self.v)

    @staticmethod
    def of(x):
        return x if isinstance(x, E) else E(torch.as_tensor(x).double())

    def _r(self, v, e, u=U32):                       # one correctly rounded fp32 operation
        return E(v, e + u * v.abs() + TINY)

    def __add__(self, o):
        o = E.of(o)
        return self._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = E.of(o)
        return self._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return E.of(o) - self

    def __neg__(self):
        return E(-self.v, self.e)

    def __mul__(self, o):
        o = E.of(o)
        return self._r(self.v * o.v, self.e * o.v.abs() + o.e * self.v.abs())

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E.of(o)
        q = self.v / o.v
        return self._r(q, (self.e + q.abs() * o.e) / o.v.abs())

    def __rtruediv__(self, o):
        return E.of(o) / self

    def __getitem__(self, k):
        return E(self.v[k], self.e[k])

    def abs(self):
        return E(self.v.abs(), self.e)

    def where(self, m, other):
        o = E.of(other)
        return E(torch.where(m, self.v, o.v), torch.where(m, self.e, o.e))


def _fn(a, v, dv, ulps):
    """a transcendental: propagated |f'(a)| e_a plus `ulps` ulp of the result (ulps may be a tensor)"""
    return E(v, dv.abs() * a.e + ulps * ULP * v.abs() + ulps * TINY)


def expf(a, ulps=ULPS["exp"]):
    v = torch.exp(a.v)
    return _fn(a, v, v, ulps)


def fast_expf(a):
    """__expf: ex2.approx of x log2 e, 2 + floor(|1.173 x|) ulp"""
    return expf(a, 2.0 + torch.floor((1.173 * a.v).abs()))


def tanhf(a):
    v = torch.tanh(a.v)
    return _fn(a, v, 1.0 - v * v, ULPS["tanh"])


def logf(a):
    return _fn(a, torch.log(a.v), 1.0 / a.v, ULPS["log"])


def log1pf(a):
    return _fn(a, torch.log1p(a.v), 1.0 / (1.0 + a.v), ULPS["log1p"])


def erff(a):
    return _fn(a, torch.erf(a.v), 2.0 / math.sqrt(math.pi) * torch.exp(-a.v * a.v), ULPS["erf"])


def rsqrtf(a):
    v = torch.rsqrt(a.v)
    return _fn(a, v, 0.5 * v / a.v, ULPS["rsqrt"])


def sqrtf(a):
    v = torch.sqrt(a.v)
    return E(v, 0.5 / v.clamp_min(1e-300) * a.e + U32 * v + TINY)


def esum(t, dim, chain):
    """a sum whose longest addition chain is `chain`: sum e + chain U32 sum |v|"""
    return E(t.v.sum(dim), t.e.sum(dim) + chain * U32 * t.v.abs().sum(dim))


def f32(x):
    return torch.as_tensor(x, dtype=torch.float32)


# ---- addition chains --------------------------------------------------------------------------------------------------
WARP = 5                                    # warp_sum: 5 butterfly levels
BLOCK = 10                                  # block_sum: a warp butterfly, then one over the warp sums


def os_chain(S):
    """ordered_sum over S partials: lane ty adds ceil(S / 16) of them, the 16 lanes are added in order, then dst += t"""
    return cdiv(S, OS_LANES) + OS_LANES + 1


def ln_row_chain(C):
    """warp-per-row LayerNorm (and, since they agree, the block kernel): lane l adds channels l, l + 32, ..., then warp_sum"""
    return cdiv(C, 32) + WARP


def ln_bwd_geometry(rows):
    """evk_layernorm_bwd / _drop_bwd: rows_per_block = max(8, ceil(rows / 528)), S = ceil(rows / rpb) blocks"""
    rpb = max(8, cdiv(rows, NUM_SMS * 4))
    return rpb, cdiv(rows, rpb)


def ln_param_chain(rows):
    """dgamma / dbeta: a lane adds its warp's rows (every 8th of the block's rpb), 8 warps add into shared memory in order,
    ordered_sum adds the S blocks"""
    rpb, S = ln_bwd_geometry(rows)
    return cdiv(rpb, 8) + 8 + os_chain(S)


def colsum_geometry(rows, n):
    """evk_colsum: want = ceil(132 * 8 / nb) row blocks, rpb = max(64, ceil(rows / want)), S = ceil(rows / rpb)"""
    nb = cdiv(n, 32)
    want = cdiv(NUM_SMS * 8, nb)
    rpb = max(64, cdiv(rows, want))
    return rpb, cdiv(rows, rpb)


def colsum_chain(rows, n):
    rpb, S = colsum_geometry(rows, n)
    return cdiv(rpb, 8) + 8 + os_chain(S)


def grid_reduce_chain(n, cap_blocks):
    """a grid-stride loop of 256-thread blocks, capped at cap_blocks, a block_sum per block and ordered_sum over the blocks"""
    G = max(1, min(cap_blocks, cdiv(n, 256)))
    return cdiv(n, G * 256) + BLOCK + 1 + os_chain(G)


G1_CAP = NUM_SMS * 16                       # vq_loss_optim.cu g1 (reduce losses, KL, AdamW) and ce_bwd
GRID1D_CAP = NUM_SMS * 32                   # elementwise.cu grid1d
SINEPOS_ADD_CAP, SINEPOS_BWD_CAP = NUM_SMS * 8, NUM_SMS * 4
OS_TRIP = NUM_SMS * 16 * 32                 # ordered_sum outputs per grid-stride trip


# ---- LayerNorm ----------------------------------------------------------------------------------------------------------
def layernorm_fwd(t, gamma, beta, eps, chain):
    """t: E [rows, C] (x, or x + res as the kernel formed it).  -> (y, mean, rstd)"""
    C = t.v.shape[-1]
    mean = esum(t, -1, chain) / float(C)
    d = t - E(mean.v[:, None], mean.e[:, None])
    var = esum(d * d, -1, chain) / float(C)
    rstd = rsqrtf(var + float(f32(eps)))
    y = d * E(rstd.v[:, None], rstd.e[:, None]) * E.of(gamma.double()) + E.of(beta.double())
    return y, mean, rstd


def ln_input(x, res=None, mask=None):
    """x (+ res) (* mask) as the kernels form it: one rounding per operation"""
    t = E.of(x.double())
    if res is not None:
        r = E.of(res.double())
        if mask is not None:
            r = r * E.of(mask.double())
        t = t + r
    return t


def layernorm_bwd(t, gamma, mean, rstd, dy, row_chain, param_chain):
    """with the kernel's own stats (mean, rstd: fp32 inputs): dx [rows, C], dgamma, dbeta"""
    C = t.v.shape[-1]
    h = (t - E.of(mean.double()[:, None])) * E.of(rstd.double()[:, None])
    d = E.of(dy.double())
    g = d * E.of(gamma.double())
    s1 = esum(g, -1, row_chain) / float(C)
    s2 = esum(g * h, -1, row_chain) / float(C)
    dx = E.of(rstd.double()[:, None]) * (g - E(s1.v[:, None], s1.e[:, None]) - h * E(s2.v[:, None], s2.e[:, None]))
    return dx, esum(d * h, 0, param_chain), esum(d, 0, param_chain)


# ---- element-wise -------------------------------------------------------------------------------------------------------
def sigmoidf_(a):
    return 1.0 / (1.0 + fast_expf(-a))


def softplusf_(a):
    sp = log1pf(expf(a))
    big = a.v > 20.0
    return E(torch.where(big, a.v, sp.v), torch.where(big, a.e, sp.e))


def unary(op, alpha, x):
    a, alpha = E.of(x.double()), float(f32(alpha))
    if op == 0:
        return a * alpha
    if op == 1:
        return a.where(a.v > 0, a * alpha)
    if op == 2:
        return tanhf(a)
    if op == 3:
        return a * tanhf(softplusf_(a))
    if op == 6:
        return 0.5 * a * (1.0 + erff(a * float(f32(0.70710678118654752))))
    return E(a.v.clamp_min(0.0))


def unary_bwd(op, alpha, x, dy):
    a, g, alpha = E.of(x.double()), E.of(dy.double()), float(f32(alpha))
    if op == 0:
        return g * alpha
    if op == 1:
        return (g * alpha).where(a.v <= 0, g)
    if op == 2:
        t = tanhf(a)
        return g * (1.0 - t * t)
    if op == 3:
        t = tanhf(softplusf_(a))
        return g * (t + a * (1.0 - t * t) * sigmoidf_(a))
    if op == 5:
        return g * (1.0 - a * a)
    return E(torch.where(a.v > 0, g.v, torch.zeros_like(g.v)))


def wn_gate(ta, sa):
    return tanhf(ta) * sigmoidf_(sa)


def wn_gate_bwd(ta, sa, d):
    t, s = tanhf(ta), sigmoidf_(sa)
    return d * s * (1.0 - t * t), d * t * s * (1.0 - s)


def glu_res(x, h1, h2):
    y = E.of(h1.double()) * sigmoidf_(E.of(h2.double()))
    return y if x is None else E.of(x.double()) + y


def glu_res_bwd(h1, h2, dy):
    s, d = sigmoidf_(E.of(h2.double())), E.of(dy.double())
    return d * s, d * E.of(h1.double()) * s * (1.0 - s)


def time_mask(B, T, lens):
    """[B * T] bool: frame t of item b is inside its length"""
    return (torch.arange(T)[None, :] < torch.as_tensor(lens)[:, None]).reshape(-1)


# ---- losses, optimiser ----------------------------------------------------------------------------------------------------
def reduce_loss(kind, a, b, scale):
    """sum over the elements of (1 - a)^2, a^2 or |a - b|, times scale, as one ordered_sum total"""
    A = E.of(a.double())
    t = (1.0 - A) * (1.0 - A) if kind == 0 else A * A if kind == 1 else (A - E.of(b.double())).abs()
    n = a.numel()
    G = max(1, min(G1_CAP, cdiv(n, 256)))
    s = esum(t, 0, cdiv(n, G * 256) + BLOCK)
    return s * scale, G


def kl_terms(zp, lq, mp, lp):
    d = E.of(zp.double()) - E.of(mp.double())
    L = E.of(lp.double())
    return (L - E.of(lq.double())) - 0.5 + 0.5 * d * d * fast_expf(L * -2.0)


def kl_bwd(zp, lq, mp, lp, gout, gscale):
    """-> dz_p, dm_p, dlogs_q, dlogs_p with g = gout * gscale (one fp32 product)"""
    g64 = float(f32(gout)) * float(f32(gscale))
    g = E(torch.tensor(g64), U32 * abs(g64))
    d = E.of(zp.double()) - E.of(mp.double())
    e = fast_expf(E.of(lp.double()) * -2.0)
    a = g * d * e
    return a, -a, E(torch.full_like(d.v, -g64), U32 * abs(g64)), g * (1.0 - d * d * e)


def adamw_step(p, g, m, v, lr, step, lr_scale, b1, b2, eps, wd, grad_scale):
    """one evk_adamw_flat update in the kernel's order; p, m, v are E (carried across steps), g an fp32 tensor"""
    lrs = E.of(torch.tensor(float(f32(lr)))) * float(f32(lr_scale))
    bc1 = E(torch.tensor(1.0 - float(f32(b1)) ** step)); bc1 = E(bc1.v, U32 * bc1.v.abs())
    bc2 = E(torch.tensor(1.0 - float(f32(b2)) ** step)); bc2 = E(bc2.v, U32 * bc2.v.abs())
    st, isq = lrs / bc1, rsqrtf(bc2)
    gr = E.of(g.double()) * float(f32(grad_scale))
    pp = p * (1.0 - lrs * float(f32(wd)))
    mm = m * float(f32(b1)) + (1.0 - E.of(torch.tensor(float(f32(b1))))) * gr
    vv = v * float(f32(b2)) + (1.0 - E.of(torch.tensor(float(f32(b2))))) * gr * gr
    den = sqrtf(vv) * isq + float(f32(eps))
    pp = pp - st * mm / den
    return pp, mm, vv, gr * gr


# ---- float32 emulation of the kernels' summation orders (CPU rehearsal) ------------------------------------------------
def butterfly(v):
    """warp_sum over the last axis (32 lanes): v += shfl_xor(v, o), o = 16 .. 1"""
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., torch.arange(32) ^ o]).float()
    return v


def lane_sums(x, lanes=32):
    """[..., n] -> [..., lanes]: lane l adds x[l], x[l + lanes], ... in turn (fp32)"""
    n = x.shape[-1]
    k = cdiv(n, lanes)
    xp = torch.zeros(*x.shape[:-1], k * lanes, dtype=torch.float32)
    xp[..., :n] = x
    xp = xp.view(*x.shape[:-1], k, lanes)
    s = torch.zeros(*x.shape[:-1], lanes, dtype=torch.float32)
    for i in range(k):
        s = s + xp[..., i, :]
    return s


def warp_row_sum(x):
    return butterfly(lane_sums(x))[..., 0]


def block_sum(v):
    """block_sum of 256 per-thread values [..., 256]: warp butterflies, then warp 0 over the 8 warp sums and 24 zeros"""
    w = butterfly(v.view(*v.shape[:-1], 8, 32))[..., 0]
    t = torch.zeros(*v.shape[:-1], 32, dtype=torch.float32)
    t[..., :8] = w
    return butterfly(t)[..., 0]


def ordered_sum(part, dst):
    """ordered_sum: part [S, n] -> dst [n] += (lane ty adds s = ty, ty + 16, ...; the 16 lane sums added in ty order)"""
    S = part.shape[0]
    acc = torch.zeros(OS_LANES, part.shape[1], dtype=torch.float32)
    for s in range(S):
        acc[s % OS_LANES] = acc[s % OS_LANES] + part[s]
    t = torch.zeros(part.shape[1], dtype=torch.float32)
    for k in range(OS_LANES):
        t = t + acc[k]
    return (dst + t).float()


def grid_partials(terms, cap_blocks):
    """per-block partials of a grid-stride loop of 256-thread blocks with a block_sum: [G]"""
    n = terms.numel()
    G = max(1, min(cap_blocks, cdiv(n, 256)))
    trips = cdiv(n, G * 256)
    tp = torch.zeros(trips * G * 256, dtype=torch.float32)
    tp[:n] = terms.reshape(-1)
    acc = torch.zeros(G * 256, dtype=torch.float32)
    for k in range(trips):
        acc = acc + tp[k * G * 256:(k + 1) * G * 256]
    return block_sum(acc.view(G, 256))


def emulate_layernorm_fwd(t, gamma, beta, eps, unbiased=False):
    """evk_layernorm_fwd in fp32 (the block and warp kernels agree): -> y, mean, rstd"""
    C = t.shape[-1]
    mean = (warp_row_sum(t) / C).float()
    d = (t - mean[:, None]).float()
    q = warp_row_sum((d * d).float())
    rstd = torch.rsqrt((q / (C - 1 if unbiased else C)).float() + f32(eps)).float()
    y = (((d * rstd[:, None]).float() * gamma).float() + beta).float()
    return y, mean, rstd


def emulate_layernorm_bwd(t, gamma, mean, rstd, dy, drop_lane=None):
    """evk_layernorm_bwd in fp32: dx and dgamma / dbeta through the per-warp, per-block and ordered_sum order.
    drop_lane = (block, warp, lane): that lane's dgamma partial is lost (a modelled fault)."""
    rows, C = t.shape
    h = ((t - mean[:, None]).float() * rstd[:, None]).float()
    g = (dy * gamma).float()
    s1 = (warp_row_sum(g) / C).float()
    s2 = (warp_row_sum((g * h).float()) / C).float()
    dx = (rstd[:, None] * ((g - s1[:, None]).float() - (h * s2[:, None]).float()).float()).float()
    rpb, S = ln_bwd_geometry(rows)
    part = torch.zeros(S, 2, C, dtype=torch.float32)
    dh, dd = (dy * h).float(), dy
    for blk in range(S):
        r0, r1 = blk * rpb, min(rows, blk * rpb + rpb)
        sg = torch.zeros(2, C, dtype=torch.float32)
        for w in range(8):
            ag = torch.zeros(2, C, dtype=torch.float32)
            for r in range(r0 + w, r1, 8):
                ag = (ag + torch.stack([dh[r], dd[r]])).float()
            if drop_lane is not None and drop_lane[:2] == (blk, w):
                ag[0, drop_lane[2]::32] = 0.0
            sg = (sg + ag).float()
        part[blk] = sg
    dg = ordered_sum(part[:, 0], torch.zeros(C))
    db = ordered_sum(part[:, 1], torch.zeros(C))
    return dx, dg, db


def emulate_colsum(x, base=None):
    rows, n = x.shape
    rpb, S = colsum_geometry(rows, n)
    part = torch.zeros(S, n, dtype=torch.float32)
    for blk in range(S):
        xb = x[blk * rpb:min(rows, blk * rpb + rpb)]
        acc = torch.zeros(8, n, dtype=torch.float32)
        for i in range(xb.shape[0]):
            acc[i % 8] = acc[i % 8] + xb[i]
        s = torch.zeros(n, dtype=torch.float32)
        for k in range(8):
            s = s + acc[k]
        part[blk] = s
    return ordered_sum(part, torch.zeros(n) if base is None else base)


def emulate_ce_fwd(logits, tgt):
    """lse and nll per row: warp max, lane-strided expf sums, warp_sum, mx + logf(se)"""
    mx = logits.max(-1).values
    lt = logits.gather(1, tgt[:, None])[:, 0]
    se = warp_row_sum(torch.exp((logits - mx[:, None]).float()).float())
    lse = (mx + torch.log(se).float()).float()
    return lse, (lse - lt).float()


def emulate_kl_terms(zp, lq, mp, lp):
    d = (zp - mp).float()
    e = torch.exp((-2.0 * lp).float()).float()
    return ((((lp - lq).float() - 0.5).float()) + ((((0.5 * d).float() * d).float() * e).float())).float()


def emulate_adamw(p, g, m, v, lr, step, lr_scale, b1, b2, eps, wd, grad_scale):
    lrs = f32(float(f32(lr)) * float(f32(lr_scale)))
    bc1, bc2 = f32(1.0 - float(f32(b1)) ** step), f32(1.0 - float(f32(b2)) ** step)
    st, isq = (lrs / bc1).float(), torch.rsqrt(bc2).float()
    gr = (g * f32(grad_scale)).float()
    pp = (p * (1.0 - lrs * f32(wd)).float()).float()
    mm = ((f32(b1) * m).float() + ((1.0 - f32(b1)).float() * gr).float()).float()
    vv = ((f32(b2) * v).float() + (((1.0 - f32(b2)).float() * gr).float() * gr).float()).float()
    pp = (pp - ((st * mm).float() / ((torch.sqrt(vv) * isq).float() + f32(eps)).float()).float()).float()
    return pp, mm, vv, (gr * gr).float()


# ---- comparison -----------------------------------------------------------------------------------------------------------
def outside_gate(got, ref, factor=SAFETY):
    """bool: got is not finite or |got - ref.v| > factor * ref.e (exact where ref.e == 0)"""
    got = got.double()
    return ~torch.isfinite(got) | ((got - ref.v).abs() > factor * ref.e)


def ratio(got, ref):
    """|got - ref.v| / (SAFETY * ref.e), 0 where both are 0"""
    err = (got.double() - ref.v).abs()
    gate = SAFETY * ref.e
    return torch.where(err == 0, torch.zeros_like(err), err / gate.clamp_min(1e-300))
