"""Float64 references and per-element error bounds for three fp32 training kernel groups, for
tests/test_gpu_train_elementwise.py; tests/test_cpu_train_ref.py rehearses them on the CPU against fp32 emulations of the
kernels' summation orders and against the repository's oracles.

  weight-norm packing   csrc/pack.cu          pa = tf32_rn(v g / |v|) and its backward dv, dg
  ScaledAdam            csrc/gpt_misc.cu      sadam_reduce / sadam_stats_sum / sadam_scalars / sadam_update, one step
  quantizer             csrc/vq_loss_optim.cu sgemm_nt_f32 + vq_argmax (nearest code)
                        csrc/vq_train.cu      vq_ema (+ Laplace smoothing), vq_st_fwd / _bwd, col_sum

The error model is tests/cudacore_ref.py's: a value is an E (float64 value of the operations on the fp32 inputs, first-order
bound of the fp32 result's distance from it), every correctly rounded fp32 operation adds U32 |result|, a sum adds its
longest addition chain (read from the kernel's order, written next to each function) times U32 sum |term|, and the gate is
SAFETY x model.  Constants the kernels form in double and round to float once carry U32 |value|.
"""
import math

import torch

from tests.cudacore_ref import BLOCK, E, F64, NUM_SMS, U32, WARP, cdiv, esum, f32, os_chain, sqrtf

TF32_REL = 2.0 ** -11            # cvt.rna.tf32.f32: half an ulp of a 10-bit mantissa, relative
PACK_THREADS = 256
SADAM_CHUNK = 8192               # train/gpt_step.py CHUNK: the chunk table's rows hold at most this many elements
SADAM_THREADS = 1024             # sadam_scalars_kernel: one 1024-thread block


def col(e):
    """E [n] -> E [n, 1]"""
    return E(e.v[:, None], e.e[:, None])


def const(x):
    """a float constant the kernel forms in double and rounds to float once"""
    return E(torch.tensor(float(x), dtype=F64), U32 * abs(float(x)))


# ---- weight norm (pack.cu) ------------------------------------------------------------------------------------------------
def pack_chain(n):
    """a row's sum: thread i adds elements i, i + 256, ... of the n = D1 Q row, then block_sum"""
    return cdiv(n, PACK_THREADS) + BLOCK


def weight_pack(v, g):
    """v fp32 [D0, n] (a torch-layout weight row-flattened: i = d1 Q + q), g fp32 [D0] or None -> E [D0, n] of
    v * (g / sqrtf(sum v^2)) before the TF32 rounding (v itself, exactly, without g)."""
    V = E.of(v.double())
    if g is None:
        return V
    ss = esum(V * V, -1, pack_chain(v.shape[1]))
    return V * col(E.of(g.double()) / sqrtf(ss))


def tf32_gate(ref, safety):
    """the extra term of a TF32-rounded result: half a TF32 ulp of the fp32 value, |w| <= |ref| + safety e"""
    return TF32_REL * (ref.v.abs() + safety * ref.e)


def weight_pack_bwd(v, g, dpa):
    """v [D0, n], g [D0], dpa [D0, n] (the packed gradient gathered into v's layout) -> (dv E [D0, n], dg E [D0]):
    nrm = sqrtf(ss), dg = dot / nrm, dv = (g / nrm) (dpa - v (dot / ss)); the cancellation inside the bracket is carried
    by the bound (its error is relative to |v dot / ss|, not to the difference)."""
    V, Dp = E.of(v.double()), E.of(dpa.double())
    chain = pack_chain(v.shape[1])
    ss = esum(V * V, -1, chain)
    dot = esum(Dp * V, -1, chain)
    nrm = sqrtf(ss)
    dg = dot / nrm
    sc, k = E.of(g.double()) / nrm, dot / ss
    return col(sc) * (Dp - V * col(k)), dg


def tf32_rna(x):
    """fp32 -> the nearest TF32 value, ties away from zero (cvt.rna.tf32.f32), as fp32"""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


# ---- ScaledAdam (gpt_misc.cu) -----------------------------------------------------------------------------------------------
def sadam_stats_chain(n):
    """sadam_reduce: a chunk of c <= 8192 elements is 256-thread strided + block_sum; sadam_stats_sum adds the tensor's
    chunks in order and then adds that to the (zero) stats entry"""
    return cdiv(min(n, SADAM_CHUNK), 256) + BLOCK + cdiv(n, SADAM_CHUNK) + 1


def sadam_step(p, g, delta, v, state, cfg, lr, gscale=1.0, as_f32=True):
    """One FlatScaledAdam.step restated per tensor in float64 with bounds, from an arbitrary injected state.
    p, g, delta, v: lists of per-tensor tensors (float32, or float64 when the restatement is run on its own);
    state: dict(step=int, rms [nt], sv [nt], sg [sup, nt], norms [period], thr [2]); cfg: SCALED_ADAM_DEFAULTS' keys.
    -> (out, decisions): out holds E values of p, delta, v (lists), rms, sv, sg, coef [nt, 2], glob [3], norms, thr and
    cs; decisions lists (what, |value - threshold|, bound) for every data-dependent branch the step took.
    The hyper-parameters reach the kernels as floats; as_f32=False keeps them in double (to compare with the oracle)."""
    F = (lambda x: float(f32(x))) if as_f32 else float
    b1, b2 = F(cfg["betas"][0]), F(cfg["betas"][1])
    clip, per, sup = F(cfg["clipping_scale"]), int(cfg["clipping_update_period"]), int(cfg["size_update_period"])
    slr, eps = F(cfg["scalar_lr_scale"]), F(cfg["eps"])
    rmin, rmax, smax = F(cfg["param_min_rms"]), F(cfg["param_max_rms"]), F(cfg["scalar_max"])
    lr, gscale = F(lr), F(gscale)
    K = lambda x: E(torch.tensor(float(x), dtype=F64))     # a constant operand, exact (E.of(float) would round it to fp32)
    step, nt = int(state["step"]), len(p)
    numel = [t.numel() for t in p]
    dec = []
    Ps = [E.of(t.double().reshape(-1)) for t in p]
    Gs = [E.of(t.double().reshape(-1)) * K(gscale) for t in g]
    # sadam_reduce + sadam_stats_sum
    pp = [esum(P * P, 0, sadam_stats_chain(n)) for P, n in zip(Ps, numel)]
    pg = [esum(P * G, 0, sadam_stats_chain(n)) for P, G, n in zip(Ps, Gs, numel)]
    gg = [esum(G * G, 0, sadam_stats_chain(n)) for G, n in zip(Gs, numel)]
    rms = [E.of(state["rms"][t].double()) for t in range(nt)]
    sv = [E.of(state["sv"][t].double()) for t in range(nt)]
    sg = [[E.of(state["sg"][k, t].double()) for t in range(nt)] for k in range(sup)]
    norms = [E.of(x) for x in state["norms"].double()]
    thr = [E.of(x) for x in state["thr"].double()]
    # sadam_scalars: step-0 rms init, then the gradient norm: thread i adds tensors i, i + 1024, ..., then block_sum
    if step == 0:
        rms = [sqrtf(pp[t] / float(numel[t])) if numel[t] > 1 else rms[t] for t in range(nt)]
    terms = [(rms[t] * rms[t] if numel[t] > 1 else E(torch.tensor(1.0, dtype=F64))) * gg[t] for t in range(nt)]
    tot = esum(E(torch.stack([x.v for x in terms]), torch.stack([x.e for x in terms])), 0, cdiv(nt, SADAM_THREADS) + BLOCK)
    cs = E(torch.tensor(1.0, dtype=F64))
    if clip > 0 and step > 0:
        tot_norm = sqrtf(tot)
        slot = step % per
        norms[slot] = tot_norm
        if step % per == 0:
            # bitonic sort of the `per` norms: exact, so only the new norm's position can move -- it must sit farther
            # from every other norm than its bound
            others = torch.stack([norms[j].v for j in range(per) if j != slot]) if per > 1 else torch.zeros(0, dtype=F64)
            if others.numel():
                dec.append(("new norm vs the other norms (sort position)", float((others - tot_norm.v).abs().min()),
                            float(tot_norm.e)))
            vals = torch.stack([x.v for x in norms])
            order = torch.argsort(vals, stable=True)
            idx = min(per - 1, (per // 4) * 2)
            thr = [E.of(torch.tensor(clip, dtype=F64)) * norms[int(order[idx])], E(torch.tensor(1.0, dtype=F64))]
        if step >= per and float(thr[1].v) != 0.0:
            ratio = thr[0] / (tot_norm + 1e-20)
            dec.append(("clipping ratio vs 1", abs(float(ratio.v) - 1.0), float(ratio.e)))
            if float(ratio.v) < 1.0:
                cs = ratio
    slot = step % sup
    coef = []
    for t in range(nt):
        if numel[t] > 1:
            sg[slot][t] = cs * pg[t]
            sstep = E(torch.tensor(0.0, dtype=F64))
            if slot == sup - 1:
                r = sqrtf(pp[t] / float(numel[t]))
                rms[t] = r
                if step > 0:
                    b2c = b2 ** sup
                    msq, ssum = E(torch.tensor(0.0, dtype=F64)), E(torch.tensor(0.0, dtype=F64))
                    for k in range(sup):
                        msq = msq + sg[k][t] * sg[k][t]
                        ssum = ssum + sg[k][t]
                    msq = msq / float(sup)
                    nv = sv[t] * const(b2c) + msq * const(1.0 - b2c)
                    sv[t] = nv
                    bc = 1.0 - b2c ** ((step + 1) // sup)
                    lslr = K(lr) * K(slr)
                    sstep = -lslr * const(math.sqrt(bc)) * ssum / (sqrtf(nv) + K(eps))
                    dec.append((f"tensor {t} rms vs param_min_rms", abs(float(r.v) - rmin), float(r.e)))
                    dec.append((f"tensor {t} rms vs param_max_rms", abs(float(r.v) - rmax), float(r.e)))
                    if float(r.v) < rmin:
                        sstep = E(torch.tensor(0.0, dtype=F64))
                    if float(r.v) > rmax:
                        sstep = -lslr * float(sup)
            if float(rms[t].e) > 0:
                dec.append((f"tensor {t} rms vs param_min_rms (fmaxf)", abs(float(rms[t].v) - rmin), float(rms[t].e)))
            mx = rms[t] if float(rms[t].v) >= rmin else E(torch.tensor(rmin, dtype=F64))
            one_b1 = 1.0 - E.of(torch.tensor(b1, dtype=F64))
            coef.append((E(torch.tensor(-lr, dtype=F64)) * one_b1 * mx, sstep * one_b1))
        else:
            lslr = K(lr) * K(slr)
            coef.append((-lslr * (1.0 - E.of(torch.tensor(b1, dtype=F64))), E(torch.tensor(0.0, dtype=F64))))
    bc2 = 1.0 - b2 ** (step + 1)
    dec.append(("bc2 vs 0.99 (double)", abs(bc2 - 0.99), 1e-12))
    glob = [const(1.0 / bc2) if bc2 < 0.99 else E(torch.tensor(1.0, dtype=F64)), const(1.0 / bc2), cs]
    # sadam_update, per element
    outp, outd, outv = [], [], []
    for t in range(nt):
        alpha, sstep = coef[t]
        scalar = numel[t] == 1
        vs = glob[1] if scalar else glob[0]
        P, G = Ps[t], Gs[t]
        d = E.of(delta[t].double().reshape(-1)) * K(b1)
        if not scalar:
            d = d + sstep * P
        vv = E.of(v[t].double().reshape(-1)) * K(b2) + (1.0 - E.of(torch.tensor(b2, dtype=F64))) * G * G
        d = d + alpha * G / (sqrtf(vv * vs) + K(eps))
        if scalar:
            dec.append((f"tensor {t} scalar vs +-scalar_max", float((P.v.abs() - smax).abs().min()), float(P.e.max())))
            P = E(P.v.clamp(-smax, smax), P.e)
        outp.append(P + d); outd.append(d); outv.append(vv)
    stack = lambda xs: E(torch.stack([x.v for x in xs]), torch.stack([x.e for x in xs]))
    out = dict(p=outp, delta=outd, v=outv, rms=stack(rms), sv=stack(sv), sg=E(torch.stack([stack(r).v for r in sg]),
               torch.stack([stack(r).e for r in sg])), coef=E(torch.stack([torch.stack([a.v, b.v]) for a, b in coef]),
               torch.stack([torch.stack([a.e, b.e]) for a, b in coef])), glob=stack(glob), norms=stack(norms),
               thr=stack(thr), cs=cs, step=step + 1)
    return out, dec


# ---- nearest code (vq_loss_optim.cu) ------------------------------------------------------------------------------------------
def sgemm_nt(a, b):
    """C = A B^T; each output is one thread's fmaf chain over k = 0 .. K-1 in order: the products are exact, the chain
    is K additions"""
    A, B = a.double(), b.double()
    K = a.shape[1]
    return E(A @ B.t(), K * U32 * (A.abs() @ B.abs().t()))


def vq_dist(x, embed, dots=None):
    """-dist[r][k] = -((|x_r|^2 - 2 dot[r][k]) + |e_k|^2) as vq_argmax forms it: |x_r|^2 256-thread strided + block_sum,
    |e_k|^2 lane-strided + warp_sum (rownorm_sq_kernel); dots from sgemm_nt (E) unless given"""
    D = x.shape[1]
    X, Em = E.of(x.double()), E.of(embed.double())
    xx = esum(X * X, -1, cdiv(D, 256) + BLOCK)
    en = esum(Em * Em, -1, cdiv(D, 32) + WARP)
    dt = sgemm_nt(x, embed) if dots is None else dots
    t = (col(xx) - 2.0 * dt) + E(en.v[None, :], en.e[None, :])
    return -t


def first_argmax(v):
    """[rows, K] -> the lowest index of each row's maximum (torch.max's tie rule)"""
    m = v.max(-1, keepdim=True).values
    K = v.shape[-1]
    idx = torch.where(v == m, torch.arange(K).expand_as(v), torch.full_like(v, K, dtype=torch.long))
    return idx.min(-1).values


# ---- trainable quantizer (vq_train.cu) ---------------------------------------------------------------------------------------
def vq_ema(x, codes, rows_ref, cluster_size, embed_avg, decay, eps):
    """x fp32 [B, T2, D], codes [B, T2]; rows t < rows_ref take part.  Per code: its rows' sum in row order (a chain of
    count additions); cs <- cs decay + (1 - decay) count, ea <- ea decay + (1 - decay) sum; then Laplace smoothing with
    sum(cs) 256-thread strided + block_sum: embed = ea / ((cs + eps) / (sum + K eps) sum).  -> (cs, ea, embed) E."""
    B, T2, D = x.shape
    K = cluster_size.shape[0]
    tr = min(rows_ref, T2)
    xs = x[:, :tr].reshape(-1, D).double()
    cd = codes[:, :tr].reshape(-1)
    oh = torch.nn.functional.one_hot(cd, K).double()                     # [n, K]
    count = oh.sum(0)
    acc = E(oh.t() @ xs, count[:, None] * U32 * (oh.t() @ xs.abs()))
    dc = float(f32(decay))
    a = 1.0 - E.of(torch.tensor(dc, dtype=F64))
    cs = E.of(cluster_size.double()) * dc + a * E(count)
    ea = E.of(embed_avg.double()) * dc + a * acc
    s = esum(cs, 0, cdiv(K, 256) + BLOCK)
    epsf = float(f32(eps))
    norm = (cs + epsf) / (s + E(torch.tensor(float(K), dtype=F64)) * epsf) * s
    return cs, ea, ea / col(norm)


def vq_st_fwd_emulate(x, q):
    """the straight-through value x + (q - x) in fp32 on the CPU (bit for bit what the kernel computes)"""
    return (x + (q - x).float()).float()


def vq_st_geometry(n):
    """vq_st_fwd: g = min(ceil(n / 256), 132 * 8) blocks of 256 threads over the n = B T2 D elements"""
    return max(1, min(cdiv(n, 256), NUM_SMS * 8))


def vq_commit_loss(x, qst, rows_ref):
    """mean over the rows t < rows_ref of (qst - x)^2: each thread adds its grid-strided elements, block_sum per block,
    vq_mean adds the g partials 1024-thread strided + block_sum, then / N"""
    B, T2, D = x.shape
    tr = min(rows_ref, T2)
    e = (qst[:, :tr] - x[:, :tr]).float().reshape(-1)              # exact replication of the kernel's fp32 difference
    n = B * T2 * D
    G = vq_st_geometry(n)
    s = esum(E.of(e.double()) * E.of(e.double()), 0, cdiv(n, G * 256) + BLOCK + cdiv(G, 1024) + BLOCK)
    N = B * tr * D
    return s / float(N) if N > 0 else E(torch.tensor(0.0, dtype=F64))


def vq_st_bwd(dy, x, qst, rows_ref, gloss):
    """dx[b][t] = (dy[b][2t] + dy[b][2t+1]) + g (x - qst), g = gloss 2 / N, on the rows t < rows_ref; exactly 0 past them"""
    B, T2, D = x.shape
    tr = min(rows_ref, T2)
    N = B * tr * D
    g = E.of(torch.tensor(float(f32(gloss)), dtype=F64)) * 2.0 / float(N)
    d0, d1 = E.of(dy[:, 0::2].double()), E.of(dy[:, 1::2].double())
    dx = (d0 + d1) + g * (E.of(x.double()) - E.of(qst.double()))
    keep = (torch.arange(T2) < tr)[None, :, None].expand(B, T2, D)
    return E(torch.where(keep, dx.v, torch.zeros_like(dx.v)), torch.where(keep, dx.e, torch.zeros_like(dx.e)))


def col_sum_chain(rows):
    """evk_col_sum: a thread adds its column over a 64-row chunk, ordered_sum adds the S chunk sums into a zeroed output"""
    return min(rows, 64) + os_chain(cdiv(rows, 64))


def col_sum(x):
    return esum(E.of(x.double()), 0, col_sum_chain(x.shape[0]))


# ---- fp32 emulations of the kernels' orders (CPU rehearsal) -------------------------------------------------------------------
def strided_block_sum(t, threads=256):
    """[..., n] fp32 -> a `threads`-thread strided loop (thread i adds i, i + threads, ...) then block_sum"""
    from tests.cudacore_ref import block_sum, butterfly, lane_sums
    s = lane_sums(t, threads)
    if threads == 256:
        return block_sum(s)
    w = butterfly(s.view(*s.shape[:-1], threads // 32, 32))[..., 0]
    z = torch.zeros(*s.shape[:-1], 32, dtype=torch.float32)
    z[..., :threads // 32] = w
    return butterfly(z)[..., 0]


def emulate_weight_pack(v, g, round_tf32=True):
    w = v
    if g is not None:
        ss = strided_block_sum((v * v).float())
        w = (v * (g / torch.sqrt(ss)).float()[:, None]).float()
    return tf32_rna(w) if round_tf32 else w


def emulate_weight_pack_bwd(v, g, dpa):
    ss = strided_block_sum((v * v).float())
    dot = strided_block_sum((dpa * v).float())
    nrm = torch.sqrt(ss).float()
    sc, k = (g / nrm).float(), (dot / ss).float()
    return (sc[:, None] * (dpa - (v * k[:, None]).float()).float()).float(), (dot / nrm).float()


def emulate_sgemm_nt(a, b):
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
    for k in range(a.shape[1]):
        acc = (acc + (a[:, k:k + 1] * b[None, :, k]).float()).float()
    return acc


def emulate_vq_dist(x, embed):
    from tests.cudacore_ref import warp_row_sum
    xx = strided_block_sum((x * x).float())
    en = warp_row_sum((embed * embed).float())
    dots = emulate_sgemm_nt(x, embed)
    return -(((xx[:, None] - (2.0 * dots).float()).float() + en[None, :]).float())


def emulate_vq_ema(x, codes, rows_ref, cluster_size, embed_avg, decay, eps, count_all_rows=False):
    B, T2, D = x.shape
    K = cluster_size.shape[0]
    tr = T2 if count_all_rows else min(rows_ref, T2)
    xs, cd = x[:, :tr].reshape(-1, D), codes[:, :tr].reshape(-1)
    dc = f32(decay)
    a = (1.0 - dc).float()
    cs, ea = cluster_size.clone(), embed_avg.clone()
    for k in range(K):
        acc = torch.zeros(D, dtype=torch.float32)
        rows = (cd == k).nonzero()[:, 0]
        for r in rows.tolist():
            acc = (acc + xs[r]).float()
        cs[k] = ((cs[k] * dc).float() + (a * float(rows.numel())).float()).float()
        ea[k] = ((ea[k] * dc).float() + (a * acc).float()).float()
    s = strided_block_sum(cs[None, :])[0]
    epsf = f32(eps)
    norm = ((((cs + epsf).float() / (s + (f32(float(K)) * epsf).float()).float()).float()) * s).float()
    return cs, ea, (ea / norm[:, None]).float()


def emulate_col_sum(x):
    from tests.cudacore_ref import ordered_sum
    rows, C = x.shape
    S = cdiv(rows, 64)
    part = torch.zeros(S, C, dtype=torch.float32)
    for s in range(S):
        acc = torch.zeros(C, dtype=torch.float32)
        for r in range(s * 64, min(rows, s * 64 + 64)):
            acc = (acc + x[r]).float()
        part[s] = acc
    return ordered_sum(part, torch.zeros(C))


def emulate_sadam(p, g, delta, v, state, cfg, lr, gscale=1.0, median_idx=None, drop_rmax=False):
    """sadam_reduce / _stats_sum / _scalars / _update in fp32 in the kernels' orders.  median_idx and drop_rmax model
    faults of the clipping median index and of the param_max_rms override.  -> dict like sadam_step's values."""
    F = lambda x: f32(x)
    b1, b2 = F(cfg["betas"][0]), F(cfg["betas"][1])
    clip, per, sup = F(cfg["clipping_scale"]), int(cfg["clipping_update_period"]), int(cfg["size_update_period"])
    slr, eps, rmin, rmax, smax = (F(cfg[k]) for k in ("scalar_lr_scale", "eps", "param_min_rms", "param_max_rms", "scalar_max"))
    lr, gscale = F(lr), F(gscale)
    step, nt = int(state["step"]), len(p)
    numel = [t.numel() for t in p]
    P = [t.reshape(-1).float() for t in p]
    G = [(t.reshape(-1).float() * gscale).float() for t in g]
    stats = torch.zeros(nt, 3)
    for t in range(nt):
        for j, terms in enumerate(((P[t] * P[t]).float(), (P[t] * G[t]).float(), (G[t] * G[t]).float())):
            acc = torch.zeros((), dtype=torch.float32)
            for c in range(0, numel[t], SADAM_CHUNK):
                acc = (acc + strided_block_sum(terms[c:c + SADAM_CHUNK][None, :])[0]).float()
            stats[t, j] = (stats[t, j] + acc).float()
    rms, sv, sg = state["rms"].float().clone(), state["sv"].float().clone(), state["sg"].float().clone()
    norms, thr = state["norms"].float().clone(), state["thr"].float().clone()
    if step == 0:
        for t in range(nt):
            if numel[t] > 1:
                rms[t] = torch.sqrt((stats[t, 0] / float(numel[t])).float())
    terms = torch.stack([((rms[t] * rms[t]).float() if numel[t] > 1 else torch.tensor(1.0)) * stats[t, 2] for t in range(nt)]).float()
    tot = strided_block_sum(terms[None, :], SADAM_THREADS)[0]
    cs = torch.tensor(1.0)
    if clip > 0 and step > 0:
        tn = torch.sqrt(tot).float()
        norms[step % per] = tn
        if step % per == 0:
            srt = norms.sort().values
            idx = min(per - 1, (per // 4) * 2) if median_idx is None else median_idx(per)
            thr[0] = (clip * srt[min(idx, per - 1)]).float()
            thr[1] = 1.0
        if step >= per and thr[1] != 0:
            cs = torch.clamp((thr[0] / (tn + F(1e-20)).float()).float(), max=1.0)
    slot = step % sup
    coef = torch.zeros(nt, 2)
    lslr = (lr * slr).float()
    for t in range(nt):
        if numel[t] > 1:
            sg[slot, t] = (cs * stats[t, 1]).float()
            sstep = torch.tensor(0.0)
            if slot == sup - 1:
                r = torch.sqrt((stats[t, 0] / float(numel[t])).float())
                rms[t] = r
                if step > 0:
                    b2c = float(b2) ** sup
                    msq, ssum = torch.tensor(0.0), torch.tensor(0.0)
                    for k in range(sup):
                        msq = (msq + (sg[k, t] * sg[k, t]).float()).float()
                        ssum = (ssum + sg[k, t]).float()
                    msq = (msq / float(sup)).float()
                    nv = ((sv[t] * F(b2c)).float() + (msq * F(1.0 - b2c)).float()).float()
                    sv[t] = nv
                    bc = 1.0 - b2c ** ((step + 1) // sup)
                    sstep = ((((-lslr) * F(math.sqrt(bc))).float() * ssum).float() / (torch.sqrt(nv) + eps).float()).float()
                    if r < rmin:
                        sstep = torch.tensor(0.0)
                    if r > rmax and not drop_rmax:
                        sstep = (-lslr * float(sup)).float()
            coef[t, 0] = (((-lr) * (1.0 - b1).float()).float() * torch.maximum(rms[t], rmin)).float()
            coef[t, 1] = (sstep * (1.0 - b1).float()).float()
        else:
            coef[t, 0] = ((-lslr) * (1.0 - b1).float()).float()
    bc2 = 1.0 - float(b2) ** (step + 1)
    vsn = F(1.0 / bc2) if bc2 < 0.99 else torch.tensor(1.0)
    outp, outd, outv = [], [], []
    for t in range(nt):
        scalar = numel[t] == 1
        vs = F(1.0 / bc2) if scalar else vsn
        d = (delta[t].reshape(-1).float() * b1).float()
        if not scalar:
            d = (d + (coef[t, 1] * P[t]).float()).float()
        vv = ((v[t].reshape(-1).float() * b2).float() + (((1.0 - b2).float() * G[t]).float() * G[t]).float()).float()
        d = (d + ((coef[t, 0] * G[t]).float() / (torch.sqrt((vv * vs).float()) + eps).float()).float()).float()
        pv = P[t].clamp(-smax, smax) if scalar else P[t]
        outp.append((pv + d).float()); outd.append(d); outv.append(vv)
    return dict(p=outp, delta=outd, v=outv, rms=rms, sv=sv, sg=sg, coef=coef, norms=norms, thr=thr, cs=cs)
