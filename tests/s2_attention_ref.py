"""Float64 reference, per-element error bounds, an fp32 emulator and the case table of the stage-2 attention operator
(ops.attention / _AttnFn: five batched contractions through evk_gconv_fwd / evk_gconv_wgrad, the fp32 kernels of
csrc/attention.cu and evk_dropout on the probabilities), for tests/test_gpu_s2_attention_elementwise.py;
tests/test_cpu_s2_attention_ref.py rehearses them on the CPU.

The operator (attentions.py:243-292, modules.py:669-682, mrte_model.py:54-59), per batch item b and head h, band tap r of
query i belonging to key j = i + r - win:
    logits[i][j] = (q_i . k_j + [0 <= r <= 2 win] q_i . Ek[r]) * scale, -> fill where i >= qlen[b] or j >= klen[b]
    P = softmax_j(logits);  Pd = P * keep / (1 - p);  band[i][r] = Pd[i][i + r - win] (0 outside [0, Tk))
    out_i = sum_j Pd[i][j] v_j + sum_r band[i][r] Ev[r]
A filled logit passes no gradient (masked_fill), so a dead query row (uniform 1/Tk with fill = -1e4) has dq = 0 and adds
nothing to dk, dEk.

Error model.  q, k, v and dout are small integers and Ek, Ev small integers times a power of two (exact_ref.ints), so
q.k, q.Ek and dout.v are exact fp32 values in every kernel family; generic (normal) operands add the bracketed terms.
Every rounding is named once:
  - [generic: the A operand q / dout, cvt.rna                                                  U_A (mode);
     the B operand K, V, V^T, K^T: cvt.rna on mma.sync, truncated by the tensor core on gconv_tc U_B (mode, family);
     one truncating accumulation per term of q.k; the fp32 FMA chain of relk_logits, the add]   U_ACC, U32 per term
  - the fp32 multiply by scale, the fp32 difference from the row maximum                         U32 per operation
  - __expf: ex2.approx after an fp32 multiply by log2e                                          U_EXP + |x| U32, relative
  - the fp32 row sum (ceil(Tk / block) serial adds per thread, two 5-step shuffle trees)        U32 per level
  - 1 / sum and the multiply by it, the multiply by 1 / (1 - p)                                 U32 per operation
  - the A operands Pd and dS, cvt.rna (hi + lo residual under 3xTF32)                           U_A (mode)
  - the tensor core's fp32 accumulation: at most one truncation per added term                  U_ACC per term
  - the fp32 FMA chains of relv_out / relk_dq over the 2 win + 1 taps, and their += into out/dq U32 per term
  - the fp32 dot sum_j P dP of attn_softmax_bwd (as the row sum), and P * (dP - dot) * scale     U32 per operation
  - the ordered fp32 partial sums of gconv_w_sum (at most 8 ceil(Tq / 256) partials and the +=) U32 per partial
  - rel_dE: an fp32 FMA chain over 32 rows per chunk, then ordered_sum over the chunks          U32 per term / chunk
Every bound below ("model") is the first-order propagation of these, evaluated in float64 from absolute values; the
gate is SAFETY (attention_ref.SAFETY = 2, justified there) times the model and no constant comes from a measurement.
Exact by construction and required bit-exact: a probability whose float64 value is 0 (fill = -inf, or fill = -1e4
beside a visible key: __expf of an argument below -104 is 0.0), a dropped probability, and every gradient through one.
"""
import numpy as np
import torch

from tests import attention_ref as A
from tests import exact_ref

U32, U_ACC, SAFETY = A.U32, A.U_ACC, A.SAFETY
U_EXP = 2.0 ** -22
# relative error of an operand as the tensor core multiplies it.  A: cvt.rna.  B: cvt.rna on the mma.sync kernels, raw
# fp32 bits (truncation) on gconv_tc_kernel.  3xTF32 (evk_set_precise(1)) runs every contraction on mma.sync with hi + lo.
MODES = {"tf32": dict(UA=2.0 ** -11, UB={"fwd_mma_sync": 2.0 ** -11, "fwd_gconv_tc": 2.0 ** -10}),
         "3xtf32": dict(UA=2.0 ** -22, UB={"fwd_mma_sync": 2.0 ** -21, "fwd_gconv_tc": 2.0 ** -21})}
PROB_FLOOR = A.PROB_FLOOR
RQ, RE = 2, 1                        # value ranges of q / k / v / dout and of Ek / Ev (before the power of two)
EK_EXP, EV_EXP = -3, -2              # Ek = ints * 2^-3, Ev = ints * 2^-2
DE_CHUNK = 32                        # rows per rel_dE block (csrc/attention.cu rpb)
G1_CAP = 132 * 32 * 256              # elements one pass of a g1() grid covers (kNumSMs * 32 blocks of 256 threads)
FAULTS = ("band shifted by one", "key klen admitted", "dead query rows not filled", "boundary drelk taps not zeroed",
          "last rel_dE chunk dropped", "backward mask differs in one float4 group", "band taken from P", "1/(1-p) applied twice")


def softmax_block(Tk):
    return 256 if Tk >= 256 else (128 if Tk >= 128 else 64)


def sum_depth(Tk):
    """fp32 additions on the path of one term of a block-wide sum: serial adds per thread, then two shuffle trees"""
    return -(-Tk // softmax_block(Tk)) + 10


# ---- layout helpers -----------------------------------------------------------------------------------------------------
def heads(x, H):
    """[B, T, H dk] -> [B, H, T, dk]"""
    B, T, C = x.shape
    return x.reshape(B, T, H, C // H).permute(0, 2, 1, 3)


def unheads(x):
    B, H, T, dk = x.shape
    return x.permute(0, 2, 1, 3).reshape(B, T, H * dk)


def band_index(Tq, Tk, win, device, shift=0):
    """key j = i + r - win of tap r of query i, and whether it lies in [0, Tk)"""
    j = torch.arange(Tq, device=device)[:, None] + torch.arange(2 * win + 1, device=device)[None, :] - win + shift
    return j, (j >= 0) & (j < Tk)


def to_band(M, win, shift=0):
    """[B, H, Tq, Tk] -> [B, H, Tq, 2 win + 1]: M[i][i + r - win], 0 outside"""
    Tq, Tk = M.shape[-2:]
    j, ok = band_index(Tq, Tk, win, M.device, shift)
    return torch.gather(M, 3, j.clamp(0, Tk - 1).expand(*M.shape[:2], -1, -1)) * ok


def from_band(Bd, Tk, win, shift=0):
    """the transpose of to_band: [B, H, Tq, 2 win + 1] -> [B, H, Tq, Tk]"""
    Tq = Bd.shape[-2]
    j, ok = band_index(Tq, Tk, win, Bd.device, shift)
    out = torch.zeros(*Bd.shape[:3], Tk, dtype=Bd.dtype, device=Bd.device)
    return out.scatter_add_(3, j.clamp(0, Tk - 1).expand(*Bd.shape[:2], -1, -1), Bd * ok)


def visible(B, Tq, Tk, qlen, klen, device):
    """[B, 1, Tq, Tk] bool: logit (i, j) is not filled"""
    vis = torch.ones(B, 1, Tq, Tk, dtype=torch.bool, device=device)
    if qlen is not None:
        vis &= (torch.arange(Tq, device=device)[None, :] < torch.as_tensor(qlen, device=device)[:, None])[:, None, :, None]
    if klen is not None:
        vis &= (torch.arange(Tk, device=device)[None, :] < torch.as_tensor(klen, device=device)[:, None])[:, None, None, :]
    return vis


def drop_inv(p):
    """the kernel's fp32 1 / (1 - p)"""
    return A.fp32(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


# ---- dropout mask of evk_dropout ------------------------------------------------------------------------------------------
def u32_to_unit(x):
    """evk_common.cuh: (x >> 8) * 2^-24, exact in fp32 and in float64"""
    return (np.asarray(x, dtype=np.uint64) >> np.uint64(8)).astype(np.float64) / 16777216.0


def keep_mask(seed, offset, sid, shape_padded, p):
    """bool [Z, Tq, ldS]: the keep flags evk_dropout draws on the pitch-padded probability buffer.  Flat element
    e = 4 i + k uses word k of Philox(seed)(offset + i, sid) and is kept iff u32_to_unit(word) >= fp32(p)."""
    n = int(np.prod(shape_padded))
    ctr = np.arange((n + 3) // 4, dtype=np.uint64) + np.uint64(offset)
    words = np.stack([np.asarray(w, dtype=np.uint64) for w in A.philox(int(seed), ctr, int(sid))], -1).reshape(-1)[:n]
    return torch.from_numpy((u32_to_unit(words) >= float(np.float32(p))).reshape(shape_padded))


# ---- float64 reference --------------------------------------------------------------------------------------------------
def attention_f64(q, k, v, Ek, Ev, H, win, scale, fill, qlen, klen, keep=None, p=0.0, dout=None):
    """q [B, Tq, C], k, v [B, Tk, C], Ek, Ev [2 win + 1, dk] (win None: no relative terms), keep bool [B, H, Tq, Tk].
    -> dict of float64 tensors: out [B, Tq, C]; logits, P, Pd [B, H, Tq, Tk]; band [B, H, Tq, 2 win + 1]; with dout also
    dq, dk, dv, dEk, dEv and the backward's intermediates (dP, dS, drel).  scale is the kernels' fp32 value."""
    B, Tq, _ = q.shape
    Tk = k.shape[1]
    sc = A.fp32(scale)
    qh, kh, vh = heads(q, H), heads(k, H), heads(v, H)
    vis = visible(B, Tq, Tk, qlen, klen, q.device)
    s = qh @ kh.transpose(-1, -2)
    if win is not None:
        s = s + from_band(qh @ Ek.t(), Tk, win)
    logits = (s * sc).masked_fill(~vis, fill)
    P = torch.softmax(logits, -1)
    ks = None if keep is None else keep.to(q.device).double() * drop_inv(p)
    Pd = P if ks is None else P * ks
    oh = Pd @ vh
    band = None
    if win is not None:
        band = to_band(Pd, win)
        oh = oh + band @ Ev
    r = dict(out=unheads(oh), logits=logits, P=P, Pd=Pd, band=band, vis=vis, ks=ks)
    if dout is None:
        return r
    doh = heads(dout, H)
    dPd = doh @ vh.transpose(-1, -2)
    if win is not None:
        dPd = dPd + from_band(doh @ Ev.t(), Tk, win)
        r["dEv"] = torch.einsum("bhir,bhid->rd", band, doh)
    dP = dPd if ks is None else dPd * ks
    dot = (P * dP).sum(-1, keepdim=True)
    dS = P * (dP - dot) * sc * vis
    dqh = dS @ kh
    if win is not None:
        drel = to_band(dS, win)
        dqh = dqh + drel @ Ek
        r.update(drel=drel, dEk=torch.einsum("bhir,bhid->rd", drel, qh))
    r.update(dq=unheads(dqh), dk=unheads(dS.transpose(-1, -2) @ qh), dv=unheads(Pd.transpose(-1, -2) @ doh), dP=dP, dS=dS,
             dot=dot)
    return r


# ---- bounds ---------------------------------------------------------------------------------------------------------------
def model(r, q, k, v, Ek, Ev, H, win, scale, mode, dout=None, p=0.0, generic=None):
    """First-order error bound of every output of `r` (attention_f64).  generic: None for the exact integer operands, or
    the kernel family ("fwd_gconv_tc" / "fwd_mma_sync") that multiplies normal q, k, v -- forward only."""
    UA = MODES[mode]["UA"]
    UB = 0.0 if generic is None else MODES[mode]["UB"][generic]
    UAg = 0.0 if generic is None else UA
    sc = A.fp32(scale)
    P, Pd, vis = r["P"], r["Pd"], r["vis"]
    B, _, Tq, Tk = P.shape
    W = 0 if win is None else 2 * win + 1
    aq, ak, av = heads(q.abs(), H), heads(k.abs(), H), heads(v.abs(), H)
    dk_ = aq.shape[-1]
    depth = sum_depth(Tk)
    live = P > 0
    t = torch.where(live, r["logits"], torch.zeros_like(P))
    Et = U32 * t.abs()
    if generic is not None:
        qk = aq @ ak.transpose(-1, -2)
        Es = (UAg + UB + dk_ * U_ACC) * qk
        if win is not None:
            Es = Es + from_band(dk_ * U32 * (aq @ Ek.abs().t()), Tk, win) + U32 * (t.abs() / sc)
        Et = Et + sc * Es
    Et = Et * (live & vis)                                               # a filled logit is exact
    mx = t.masked_fill(~live, float("-inf")).amax(-1, keepdim=True)
    x = (t - mx) * live
    Ex = Et + Et.amax(-1, keepdim=True) + U32 * x.abs()
    ee = (Ex + U_EXP + x.abs() * U32) * live
    es = (P * ee).sum(-1, keepdim=True) + depth * U32
    eP = (ee + es + 2 * U32) * live                                      # relative error of P
    ud = U32 if p > 0 else 0.0
    EPd = Pd * (eP + ud)
    pv = UA + UB + Tk * U_ACC
    Eo = (EPd + Pd * pv) @ av
    m = dict(P=P * eP, Pd=EPd)
    if win is not None:
        aEk, aEv = Ek.abs(), Ev.abs()
        Eband = to_band(EPd, win)
        oh = heads(r["out"], H).abs()
        Eo = Eo + Eband @ aEv + W * U32 * (r["band"] @ aEv) + U32 * oh
        m["band"] = Eband
    m["out"] = unheads(Eo)
    if dout is None:
        return m
    assert generic is None
    ado = heads(dout.abs(), H)
    dP, dS = r["dP"], r["dS"]
    PdP = (P * dP).abs()
    Edot = (PdP * (eP + 2 * ud + U32)).sum(-1, keepdim=True) + depth * U32 * PdP.sum(-1, keepdim=True)
    EdS = (dS.abs() * (eP + 3 * U32) + P * sc * (ud * dP.abs() + Edot)) * vis
    nparts = 8 * -(-Tq // 256) + 1
    wg = UA + Tq * U_ACC + nparts * U32
    Edq = (EdS + dS.abs() * (UA + Tk * U_ACC)) @ ak
    m["dk"] = unheads((EdS + dS.abs() * wg).transpose(-1, -2) @ aq)
    m["dv"] = unheads((EPd + Pd * wg).transpose(-1, -2) @ ado)
    if win is not None:
        Edrel = to_band(EdS, win)
        adrel = r["drel"].abs()
        Edq = Edq + Edrel @ aEk + W * U32 * (adrel @ aEk) + U32 * heads(r["dq"], H).abs()
        ch = (DE_CHUNK + -(-B * H * Tq // DE_CHUNK)) * U32
        m["dEk"] = torch.einsum("bhir,bhid->rd", Edrel, aq.expand(B, H, Tq, dk_)) + ch * torch.einsum("bhir,bhid->rd", adrel, aq)
        m["dEv"] = torch.einsum("bhir,bhid->rd", Eband, ado) + ch * torch.einsum("bhir,bhid->rd", r["band"], ado)
    m["dq"] = unheads(Edq)
    return m


# ---- float32 emulation of the operator ---------------------------------------------------------------------------------
def b_operand(x, mode, family):
    """the value the tensor core multiplies for an fp32 B operand (K, V, V^T, K^T) of evk_gconv_fwd"""
    if mode == "tf32" and family == "fwd_gconv_tc":
        return (x.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double()
    return A.a_operand(x, mode)


def emulate(q, k, v, Ek, Ev, H, win, scale, fill, qlen, klen, mode, families, keep=None, p=0.0, dout=None, fault=None):
    """fp32 emulation: operands rounded by family and mode, products accumulated in float64 and rounded to fp32 once, fp32
    softmax (correctly rounded exp), fp32 relative-position chains.  `fault` names one modelled kernel fault (FAULTS).
    -> dict like attention_f64 (float64 tensors holding fp32 values)."""
    f = torch.float32
    B, Tq, _ = q.shape
    Tk = k.shape[1]
    sc = torch.tensor(A.fp32(scale), dtype=f)
    qh, kh, vh = heads(q, H), heads(k, H), heads(v, H)
    vis = visible(B, Tq, Tk, qlen, klen, q.device)
    visk = vis
    if fault == "key klen admitted":
        visk = visible(B, Tq, Tk, qlen, torch.as_tensor(klen) + 1, q.device)
    elif fault == "dead query rows not filled":
        visk = visible(B, Tq, Tk, None, klen, q.device)
    s = (A.a_operand(qh, mode) @ b_operand(kh, mode, families["qk"]).transpose(-1, -2)).float()
    if win is not None:
        rel = (qh.float().double() @ Ek.t()).float()
        s = s + from_band(rel, Tk, win, 1 if fault == "band shifted by one" else 0)
    t = (s * sc).masked_fill(~visk, fill)
    e = torch.exp(t - t.amax(-1, keepdim=True))
    P = e * (1.0 / e.sum(-1, keepdim=True))
    Pd = P
    if keep is not None:
        inv = torch.tensor(drop_inv(p), dtype=f)
        Pd = torch.where(keep, P * inv, torch.zeros((), dtype=f))
        if fault == "1/(1-p) applied twice":
            Pd = Pd * inv
    oh = (A.a_operand(Pd, mode) @ b_operand(vh, mode, families["pv"])).float()
    band = None
    if win is not None:
        band = to_band(P if fault == "band taken from P" else Pd, win)
        oh = oh + (band.double() @ Ev).float()
    r = dict(out=unheads(oh).double(), P=P.double(), Pd=Pd.double(), band=None if band is None else band.double())
    if dout is None:
        return r
    doh = heads(dout, H)
    dPd = (A.a_operand(doh, mode) @ b_operand(vh, mode, families["dov"]).transpose(-1, -2)).float()
    if win is not None:
        dPd = dPd + from_band((doh @ Ev.t()).float(), Tk, win)
        r["dEv"] = torch.einsum("bhir,bhid->rd", band.double(), doh).float().double()
    dP = dPd
    if keep is not None:
        kb = keep
        if fault == "backward mask differs in one float4 group":
            kb = keep.clone()
            kb[-1, -1, Tq // 4, 4:8] = ~kb[-1, -1, Tq // 4, 4:8]
        dP = torch.where(kb, dPd * inv, torch.zeros((), dtype=f))
    dot = (P * dP).sum(-1, keepdim=True)
    dS = torch.where(visk, P * (dP - dot) * sc, torch.zeros((), dtype=f))
    dSa = A.a_operand(dS, mode)
    dqh = (dSa @ b_operand(kh, mode, families["dsk"])).float()
    if win is not None:
        drel = to_band(dS, win)
        if fault == "boundary drelk taps not zeroed":
            drel = torch.where(band_index(Tq, Tk, win, q.device)[1], drel, torch.ones((), dtype=f))
        dqh = dqh + (drel.double() @ Ek).float()
        dr = drel.double()
        if fault == "last rel_dE chunk dropped":
            dr = dr.clone().view(-1, 2 * win + 1)
            dr[(dr.shape[0] - 1) // DE_CHUNK * DE_CHUNK:] = 0
            dr = dr.view(drel.shape)
        r["dEk"] = torch.einsum("bhir,bhid->rd", dr, qh).float().double()
    r.update(dq=unheads(dqh).double(), dk=unheads((dSa.transpose(-1, -2) @ A.a_operand(qh, mode)).float()).double(),
             dv=unheads((A.a_operand(Pd, mode).transpose(-1, -2) @ A.a_operand(doh, mode)).float()).double())
    return r


# ---- the case table -------------------------------------------------------------------------------------------------------
def _case(name, B, Tq, Tk, C, H, win=None, fill=-1e4, masks="qk", scale=None, p=0.0):
    """families: the dispatch slot (ops.DISPATCH_SLOTS) each contraction's flops land on in TF32 mode.  Q K^T and dO V^T
    contract over dk (a multiple of 4); P V and dS K over Tk, which gconv_tc_kernel takes only when Tk % 4 == 0; H > 1 or a
    per-item weight operand keeps all of them off the TMA kernel; dV and dK are weight-gradient shaped."""
    over_tk = "fwd_gconv_tc" if Tk % 4 == 0 else "fwd_mma_sync"
    fam = dict(qk="fwd_gconv_tc", pv=over_tk, dov="fwd_gconv_tc", dsk=over_tk, dv="wgrad_mma_sync", dk="wgrad_mma_sync")
    return dict(name=name, B=B, Tq=Tq, Tk=Tk, C=C, H=H, win=win, fill=fill, masks=masks,
                scale=(C // H) ** -0.5 if scale is None else scale, p=p, families=fam)


def _self(name, B, T, C=64, **kw):
    return _case(name, B, T, T, C, 2, win=4, **kw)


STYLE = dict(fill=float("-inf"), masks="k", scale=128.0 ** -0.5)
CASES = [
    # the three configurations of the stage-2 step (models.py) at a padded batch of the trainer
    _self("self step", 4, 352, C=192),
    _case("style step", 4, 352, 352, 128, 2, **STYLE),
    _case("cross step", 4, 352, 128, 512, 4),
    # softmax block sizes 64 / 128 / 256 and the strided loop past 256; Tk % 4 of 3, 0, 3, 0, 3, 0, 1
    *[_self(f"self T={T}", 2, T) for T in (63, 64, 127, 128, 255, 256, 257)],
    # both families of P V and dS K on the same queries: Tk % 4 = 0 (gconv_tc) beside 1, 2, 3 (mma.sync, padded pitch of S)
    *[_case(f"cross Tk={Tk}", 3, 96, Tk, 128, 4) for Tk in (128, 129, 130, 131)],
    _case("style Tk=130", 3, 70, 130, 128, 2, **STYLE),
    # window edges: T < win, T = win, win + 1, 2 win + 1; 3 * 2 * T rows are never a multiple of the 32-row rel_dE chunk and
    # at T = 9 the first chunk spans the head boundary at row 9 and the batch boundary at row 18
    *[_self(f"self T={T}", 3, T) for T in (1, 2, 4, 5, 9)],
    # B H Tq dk = 1179648 > G1_CAP: relk_dq / relv_out take a second grid-stride pass
    _self("self second pass", 16, 384, C=192),
]
# dropout on the probabilities: the self configuration on a padded pitch (ldS = 132 != Tk), the style one at the step shape
DROP_CASES = [c for p in (0.1, 0.5) for c in (_self(f"self drop p={p}", 2, 130, C=192, p=p),
                                             _case(f"style drop p={p}", 2, 352, 352, 128, 2, p=p, **STYLE))]
GENERIC_CASES = [_self("generic T=352", 2, 352, C=192), _self("generic T=351", 2, 351, C=192)]
DROP_SEED, DROP_TAG = 4242, "s2_attention_elementwise.drop"


def case_lens(c):
    """ragged (qlen, klen) of a case: the last item at full length, one at length 1 (B >= 3), the rest in between"""
    def lens(T, rot):
        base = [max(T - 5, 1), 1, max(T // 2, 1), T]
        n = c["B"]
        return [max(T - 7 * b, 1) for b in range(n - 4)] + [base[(b + (rot if n >= 4 else 0)) % 4] for b in range(4 - min(n, 4), 4)]
    kl = lens(c["Tk"], 0)
    if c["masks"] == "k":
        return None, kl
    return (kl if c["Tq"] == c["Tk"] and c["win"] is not None else lens(c["Tq"], 1)), kl


def case_inputs(c, seed, generic=False):
    """-> q [B, Tq, C], k, v [B, Tk, C], dout [B, Tq, C], Ek, Ev [2 win + 1, dk] or None, float64 on the CPU"""
    g = torch.Generator().manual_seed(seed)
    B, Tq, Tk, C, dk = c["B"], c["Tq"], c["Tk"], c["C"], c["C"] // c["H"]
    if generic:
        q, k, v, do = (torch.randn(B, T, C, generator=g).double() for T in (Tq, Tk, Tk, Tq))
    else:
        q, k, v, do = (exact_ref.ints((B, T, C), RQ, g) for T in (Tq, Tk, Tk, Tq))
    Ek = Ev = None
    if c["win"] is not None:
        W = 2 * c["win"] + 1
        Ek = exact_ref.ints((W, dk), RE, g) * 2.0 ** EK_EXP
        Ev = exact_ref.ints((W, dk), RE, g) * 2.0 ** EV_EXP
    return q, k, v, do, Ek, Ev


def exact_bounds(c):
    """the largest sum |a| |b| of the products that must be exact (Q K^T, dO V^T, q.Ek and dO.Ev in units of 2^EK_EXP /
    2^EV_EXP, and the sum S + rel in units of 2^EK_EXP), from the shapes and ranges alone"""
    dk = c["C"] // c["H"]
    qk = dk * RQ * RQ
    return dict(qk=qk, dov=qk, rel=dk * RQ * RE, logit=qk * 2 ** -EK_EXP + dk * RQ * RE)


def readout_heads(c):
    return -(-c["Tk"] // (c["C"] // c["H"]))


def readout_inputs(c, seed):
    """The probe of every probability: H' = ceil(Tk / dk) heads share one q, k; v of head h is the identity on key block h.
    -> q [B, Tq, H' dk], k, v [B, Tk, H' dk], q1 [B, Tq, dk], k1 [B, Tk, dk], keys [H', dk] (A.readout_keys), Ek or None"""
    g = torch.Generator().manual_seed(seed)
    B, Tq, Tk, dk = c["B"], c["Tq"], c["Tk"], c["C"] // c["H"]
    Hr = readout_heads(c)
    q1, k1 = exact_ref.ints((B, Tq, dk), RQ, g), exact_ref.ints((B, Tk, dk), RQ, g)
    Ek = None if c["win"] is None else exact_ref.ints((2 * c["win"] + 1, dk), RE, g) * 2.0 ** EK_EXP
    V = A.readout_v(Tk, Hr, dk)[None].expand(B, Tk, Hr * dk).contiguous()
    return q1.repeat(1, 1, Hr), k1.repeat(1, 1, Hr), V, A.readout_keys(Tk, Hr, dk), Ek


def gather_keys(M, keys):
    """M [B, H', Tq, Tk] -> [B, Tq, H' dk]: column h dk + c reads M[b, h, i, keys[h, c]] (0 where the key is past Tk)"""
    Hr, dk = keys.shape
    keys = keys.to(M.device)
    idx = keys.clamp(min=0)[None, :, None, :].expand(M.shape[0], Hr, M.shape[2], dk)
    return unheads(torch.gather(M, 3, idx) * (keys >= 0)[None, :, None, :])


def band_probe(win, dk):
    """Ev whose row r is the unit vector e_r: with v = 0 the output's first 2 win + 1 columns of each head are the band"""
    return torch.eye(2 * win + 1, dk, dtype=torch.float64)


# ---- gate and report -------------------------------------------------------------------------------------------------------
def outside(got, ref, bound):
    """bool per element: |got - ref| > SAFETY * bound, got not finite, or got != 0 where ref == 0 has a zero bound"""
    return A.outside_gate(got, ref.cpu(), bound.cpu())


def locate(c, what, idx):
    """the coordinates of one element of output `what` with the tile, softmax block and rel_dE chunk it falls in"""
    H, Tq, Tk = c["H"], c["Tq"], c["Tk"]
    if what in ("dEk", "dEv"):
        return f"tap r={idx[0]}, d={idx[1]} (summed over {-(-c['B'] * H * Tq // DE_CHUNK)} rel_dE chunks)"
    dk = c["C"] // H                                                     # a readout has more heads of the same width
    b, t, col = idx
    h, d = col // dk, col % dk
    s = f"b={b}, h={h}, {'j' if what in ('dk', 'dv') else 'i'}={t} (128-row tile {t // 128}), c={d}"
    if what not in ("dk", "dv"):
        s += f", softmax block {softmax_block(Tk)}, rel_dE chunk {((b * H + h) * Tq + t) // DE_CHUNK}"
    return s


def report(c, what, got, ref, bound, keys=None, limit=8):
    """None if every element is inside the gate, else the failure text listing the first mismatches"""
    got = got.detach().double().cpu()
    ref, bound = ref.cpu(), bound.cpu()
    bad = outside(got, ref, bound)
    if not bool(bad.any()):
        return None
    lines = []
    for idx in bad.nonzero()[:limit].tolist():
        where = locate(c, what, idx)
        if keys is not None:
            dk = keys.shape[1]
            where += f", key j={int(keys[idx[2] // dk, idx[2] % dk])}"
        lines.append(f"  [{where}] got {float(got[tuple(idx)])!r} want {float(ref[tuple(idx)])!r} "
                     f"gate {SAFETY * float(bound[tuple(idx)]):.3g}")
    return f"{c['name']} {what}: {int(bad.sum())} of {bad.numel()} outputs outside the gate\n" + "\n".join(lines)


def worst(got, ref, bound):
    r = A.ratio(got.detach(), ref.cpu(), bound.cpu())
    return float(r.max()) if r.numel() else 0.0
