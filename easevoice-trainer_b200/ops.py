"""Autograd operators over channels-last tensors, each a thin wrapper around libevk_sm90 kernels.

Layout: an activation is [B, T, C] fp32 with unit channel stride (row pitch = stride(-2)); column slices of a
contiguous tensor are valid operands (no copies).  Discriminator "period" views are [B, H*P, C] with the inner
width P passed explicitly.  Lengths are int32 device tensors [B].

Nothing here falls back to torch math: if the library or the GPU is missing, `lib.init()` raises.
"""
import ctypes
import os
import math

import torch

from . import lib as L

ACT_NONE, ACT_LRELU, ACT_RELU, ACT_TANH = 0, 1, 2, 3
ACT_GELU = 4             # exact erf GELU in the GEMM epilogue (forward only)
UN_SCALE, UN_LRELU, UN_TANH, UN_MISH, UN_RELU, UN_TANH_FROM_OUT, UN_GELU = 0, 1, 2, 3, 4, 5, 6

_launches = 0          # number of libevk kernel-launching calls (bench.py reports it)
USE_NVTX = os.environ.get("EVK_NVTX", "0") != "0"


class nvtx_range:
    """NVTX range around a phase of a step when EVK_NVTX=1 (off: a no-op context manager, nothing on the hot path)."""
    __slots__ = ("name",)

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if USE_NVTX:
            torch.cuda.nvtx.range_push(self.name)
        return self

    def __exit__(self, *exc):
        if USE_NVTX:
            torch.cuda.nvtx.range_pop()
        return False


def launches():
    return _launches


def _lib():
    return L.init()


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


# ---- optional per-call device timing (bench.py roofline / breakdown; off by default) -------------------------
_prof = None


def profile_begin():
    """Start recording (name, CUDA-event pair, algorithmic flops, algorithmic bytes) for every library call."""
    global _prof
    _prof = []


def profile_end():
    """-> {family: dict(calls, ms, flops, bytes)}; synchronises once at the end (never inside the step)."""
    global _prof
    rec, _prof = _prof, None
    torch.cuda.synchronize()
    agg = {}
    for name, e0, e1, fl, by in rec:
        a = agg.setdefault(name, dict(calls=0, ms=0.0, flops=0.0, bytes=0.0))
        a["calls"] += 1
        a["ms"] += e0.elapsed_time(e1)
        a["flops"] += fl
        a["bytes"] += by
    return agg


DISPATCH_SLOTS = ("fwd_gemm_tma", "fwd_gconv_tc", "fwd_mma_sync", "fwd_direct", "wgrad_gemm_tma", "wgrad_mma_sync", "wgrad_direct",
                  "gemm_tf32", "fwd_gemv")


def dispatch_reset():
    L.check(_lib().evk_dispatch_stats_reset())


def dispatch_stats():
    """-> {kernel family: algorithmic flops enqueued since dispatch_reset()} (host-side accounting in the library)."""
    buf = (ctypes.c_double * len(DISPATCH_SLOTS))()
    L.check(_lib().evk_dispatch_stats(buf, len(DISPATCH_SLOTS)))
    return dict(zip(DISPATCH_SLOTS, [float(v) for v in buf]))


PROF_SHAPES = False        # tools/shape_profile.py: key the profile by launch shape as well as by kernel family


def _timed(name, fn, flops=0.0, nbytes=0.0, tag=None):
    if _prof is None:
        return fn()
    before = dispatch_stats() if flops else None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    if before is not None:                      # which kernel family served this contraction (library-side accounting)
        after = dispatch_stats()
        grown = [k for k in DISPATCH_SLOTS if after[k] > before[k]]
        if grown:
            name = f"{name}:{grown[0]}"
    if PROF_SHAPES and tag is not None:
        name = f"{name}|{tag}"
    _prof.append((name, e0, e1, flops, nbytes))
    return r


def _call(name, *args):
    global _launches
    _launches += 1
    _timed(name, lambda: L.check(getattr(_lib(), name)(*args, _st())))


def _call_f(name, flops, *args, tag=None):
    """_call with an algorithmic flop count attached (contractions: shows up in profile_end / the bench roofline)."""
    global _launches
    _launches += 1
    _timed(name, lambda: L.check(getattr(_lib(), name)(*args, _st())), flops, tag=tag)


def _rows(t):
    """-> (rows, C, ld) of a channels-last tensor viewed as a row matrix."""
    assert t.dtype == torch.float32 and t.is_cuda, (t.dtype, t.device)
    if t.dim() == 1:
        return 1, t.shape[0], t.shape[0]
    C = t.shape[-1]
    assert C == 1 or t.stride(-1) == 1, f"channel stride must be 1, got {t.stride()}"
    if t.dim() == 2:
        return t.shape[0], C, (t.stride(0) if t.shape[0] > 1 else max(C, t.stride(0)))
    assert t.dim() == 3
    B, T, _ = t.shape
    if T == 1:
        ld = t.stride(0) if B > 1 else C
    else:
        ld = t.stride(1)
        assert B == 1 or t.stride(0) == T * ld, f"batch stride {t.stride(0)} != T*ld {T * ld}"
    return B * T, C, ld


def _c(t):
    """contiguous channels-last (copies only when needed)."""
    return t if (t.stride(-1) == 1 or t.shape[-1] == 1) and t.is_contiguous() else t.contiguous()


def _ok_rows(t):
    try:
        _rows(t)
        return True
    except AssertionError:
        return False


def _cl(t):
    return t if _ok_rows(t) else t.contiguous()


# ------------------------------------------------------------------------------------------------
# RNG state (device resident => CUDA-graph replay safe)
# ------------------------------------------------------------------------------------------------
_rng = {}


def rng_state(device=None):
    device = device or torch.device("cuda", torch.cuda.current_device())
    key = str(device)
    if key not in _rng:
        _rng[key] = torch.tensor([1234, 0], dtype=torch.int64, device=device)
    return _rng[key]


def manual_seed(seed, device=None):
    st = rng_state(device)
    st.copy_(torch.tensor([seed, 0], dtype=torch.int64))


def advance_rng(inc=1 << 32):
    _call("evk_advance_rng", _p(rng_state()), ctypes.c_uint64(inc))


_stream_ids = {}


def stream_id(tag):
    """stable small integer per call-site tag (Philox stream selector)."""
    if tag not in _stream_ids:
        _stream_ids[tag] = len(_stream_ids) + 1
    return _stream_ids[tag]


# ------------------------------------------------------------------------------------------------
# descriptor helpers
# ------------------------------------------------------------------------------------------------
def _desc(off=(), **kw):
    """-> GconvDesc with the given fields; every other field is zero or null, except H and G, which default to 1.
    Tensors are passed by data pointer, an int pointer field as the raw device address."""
    d = L.GconvDesc(**{"H": 1, "G": 1, **{k: v.data_ptr() if isinstance(v, torch.Tensor) else v for k, v in kw.items()}})
    assert len(off) <= L.MAX_TAPS
    for i, o in enumerate(off):
        d.off[i] = int(o)
    return d


# the extra operand of an entry point, attached to the descriptor object (not C fields): wgrad's transposed dY, dgrad's PB
_DESC_EXTRA = {"evk_gconv_wgrad": ("dyt", "ld_dyt"), "evk_gconv_dgrad": ("wt", "ld_wt")}


def _run_desc(fn, d):
    """one descriptor launch; evk_gconv_wgrad / evk_gconv_dgrad also get the operand attached as d.dyt / d.wt (_DESC_EXTRA)"""
    global _launches
    _launches += 1
    flops = 2.0 * d.Z * d.J * d.P * d.N * (d.C // max(d.G, 1)) * d.Q
    extra = _DESC_EXTRA.get(fn)
    args = (getattr(d, extra[0], None), getattr(d, extra[1], 0)) if extra else ()
    _timed(fn, lambda: L.check(getattr(_lib(), fn)(ctypes.byref(d), *args, _st())), flops,
           tag=(f"Z{d.Z} J{d.J} P{d.P} C{d.C} N{d.N} Q{d.Q} s{d.is_}" if PROF_SHAPES else None))


class PackedW:
    """Operand-packed weight: pa [Q, D0, lda] (differentiable), pb [Q, D1, ldb] (derived copy)."""
    __slots__ = ("pa", "pb", "D0", "D1", "Q")

    def __init__(self, pa, pb, D0, D1, Q):
        self.pa, self.pb, self.D0, self.D1, self.Q = pa, pb, D0, D1, Q


def _pad4(n):
    return n if n < 4 else (n + 3) // 4 * 4


def _pack_geometry(v, pad0, pad1):
    """-> (D0, D1, Q, D0p, D1p, lda, ldb) of the packed operands PA [Q, D0p, lda] and PB [Q, D1p, ldb] of the torch-layout
    weight v [D0, D1, Q(,1)].  Channel dims < 4 are zero-padded to pad0 / pad1 so every conv is 16-byte tileable."""
    D0, D1 = v.shape[0], v.shape[1]
    D0p, D1p = max(D0, pad0), max(D1, pad1)
    return D0, D1, v.numel() // (D0 * D1), D0p, D1p, _pad4(D1p), _pad4(D0p)


class _PackFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v, g, need_pb, pad0, pad1):
        D0, D1, Q, D0p, D1p, lda, ldb = _pack_geometry(v, pad0, pad1)
        exact = (D0p == D0 and D1p == D1)
        pa = (torch.zeros if (lda != D1 or not exact) else torch.empty)((Q, D0p, lda), device=v.device, dtype=torch.float32)
        pb = None
        if need_pb:
            pb = (torch.zeros if (ldb != D0 or not exact) else torch.empty)((Q, D1p, ldb), device=v.device, dtype=torch.float32)
        vc = v.contiguous()
        gc = g.contiguous() if g is not None else None
        job = L.PackJob(v=_p(vc), g=_p(gc), pa=_p(pa), pb=_p(pb), D0=D0, D1=D1, Q=Q, lda=lda, D0p=D0p, ldb=ldb, D1p=D1p)
        _call("evk_weight_pack_one", ctypes.byref(job))
        ctx.save_for_backward(vc, gc)
        ctx.job = job
        if pb is None:
            pb = torch.empty(0, device=v.device)
        ctx.mark_non_differentiable(pb)
        return pa, pb

    @staticmethod
    def backward(ctx, dpa, _dpb):
        v, g = ctx.saved_tensors
        dpa = dpa.contiguous()
        dv = torch.empty_like(v)
        dg = torch.empty_like(g) if g is not None else None
        job = ctx.job
        job.dpa, job.dv, job.dg = _p(dpa), _p(dv), _p(dg)
        _call("evk_weight_pack_bwd_one", ctypes.byref(job))
        return dv, dg, None, None, None


def pack_weight(v, g=None, need_pb=True, pad0=0, pad1=0):
    """weight-norm (if g) + pack.  v: torch-layout weight [D0, D1, Q(,1)]; pad0/pad1 zero-pad the channel dims."""
    pa, pb = _PackFn.apply(v, g, need_pb, pad0, pad1)
    _, _, Q, D0p, D1p, _, _ = _pack_geometry(v, pad0, pad1)
    return PackedW(pa, pb if need_pb else None, D0p, D1p, Q)


# ---- pooled zero-initialised scratch for small accumulators (bias gradients) -------------------------------------------
# A backward pass needs ~300 tiny zero-filled vectors (one per bias): as separate torch.zeros they are 300 fill launches.
# Inside `with grad_pool():` they are slices of one persistent buffer that is cleared by ONE memset when the scope opens.
# Only for callers that consume the gradients before the next scope opens (the train steps copy them into their flat
# gradient arena right away); everything else gets ordinary torch.zeros.
class _ZeroPool:
    def __init__(self):
        self.buf, self.off, self.high, self.on = None, 0, 0, False

    def take(self, n, device):
        if not self.on:
            return torch.zeros(n, device=device, dtype=torch.float32)
        device = torch.device(device)
        if self.buf is None or self.buf.device != device:
            self.buf, self.off, self.high = torch.zeros(1 << 20, device=device, dtype=torch.float32), 0, 0
        a = (self.off + 3) // 4 * 4
        if a + n > self.buf.numel():
            return torch.zeros(n, device=device, dtype=torch.float32)
        self.off = a + n
        self.high = max(self.high, self.off)
        return self.buf[a:a + n]


_zpool = _ZeroPool()


class grad_pool:
    def __enter__(self):
        if _zpool.buf is not None and _zpool.high:
            _zpool.buf[:_zpool.high].zero_()
        _zpool.off, _zpool.on = 0, True
        return self

    def __exit__(self, *exc):
        _zpool.on = False
        return False


# ---- whole-network packing: one launch per network per step (pack.cu) ---------------------------------------------
_dpa_views = {}          # data_ptr of a packed weight -> its slice of the plan's (pre-zeroed) packed-gradient arena
_dpa_taken = set()       # slices already handed to a backward since the plan was last zeroed


def dpa_buffer(pa):
    """where a weight-gradient kernel accumulates d(pa): the plan's arena slice when pa comes from a PackPlan (zeroed once
    per step by the plan), else a fresh zero tensor.  A weight used twice in one forward (the DPO branches) gets the slice
    for its first gradient only -- autograd SUMS the gradients of the uses, so they must live in distinct buffers."""
    key = pa.data_ptr()
    v = _dpa_views.get(key)
    if v is not None and v.shape == pa.shape and key not in _dpa_taken:
        _dpa_taken.add(key)
        return v
    return torch.zeros_like(pa)


class PackPlan:
    """Static layout of every packed weight of one network.  reqs: [(key, v, g or None, need_pb, pad0, pad1, wants_grad)].
    All arenas are allocated once; the job table holds raw device pointers (parameters must already live where they will
    stay -- FlatAdamW's arena)."""

    def __init__(self, reqs, with_grad):
        dev = reqs[0][1].device
        self.reqs, self.with_grad = reqs, with_grad
        al = lambda n: (n + 63) // 64 * 64                         # 256-byte aligned regions (TMA bases need 16)
        geo, off_pa, off_pb, off_g = [], 0, 0, 0
        for key, v, g, need_pb, pad0, pad1, wants in reqs:
            D0, D1, Q, D0p, D1p, lda, ldb = _pack_geometry(v, pad0, pad1)
            geo.append((D0, D1, Q, D0p, D1p, lda, ldb, off_pa, off_pb if need_pb else -1, off_g))
            off_pa += al(Q * D0p * lda)
            if need_pb:
                off_pb += al(Q * D1p * ldb)
            off_g += al(v.numel()) + (al(g.numel()) if g is not None else 0)
        self.arena_pa = torch.zeros(off_pa, device=dev, dtype=torch.float32)
        self.arena_pb = torch.zeros(max(off_pb, 1), device=dev, dtype=torch.float32)
        self.arena_dpa = torch.zeros(off_pa, device=dev, dtype=torch.float32) if with_grad else None
        self.arena_dvg = torch.zeros(off_g, device=dev, dtype=torch.float32) if with_grad else None
        jobs = (L.PackJob * len(reqs))()
        rows, rows_bwd, row0 = [], [], 0
        self.pa, self.pb, self.dpa, self.grads, self.params, self.sig = [], [], [], [], [], []
        for i, ((key, v, g, need_pb, pad0, pad1, wants), (D0, D1, Q, D0p, D1p, lda, ldb, opa, opb, og)) in enumerate(zip(reqs, geo)):
            pa = self.arena_pa[opa:opa + Q * D0p * lda].view(Q, D0p, lda)
            pb = self.arena_pb[opb:opb + Q * D1p * ldb].view(Q, D1p, ldb) if need_pb else None
            j = jobs[i]
            j.v, j.g, j.pa, j.pb = v.data_ptr(), (g.data_ptr() if g is not None else None), pa.data_ptr(), (pb.data_ptr() if pb is not None else None)
            j.D0, j.D1, j.Q, j.lda, j.D0p, j.ldb, j.D1p, j.row0 = D0, D1, Q, lda, D0p, ldb, D1p, row0
            self.pa.append(pa); self.pb.append(pb)
            if with_grad:
                dpa = self.arena_dpa[opa:opa + Q * D0p * lda].view(Q, D0p, lda)
                dv = self.arena_dvg[og:og + v.numel()].view(v.shape)
                dg = self.arena_dvg[og + al(v.numel()):og + al(v.numel()) + g.numel()].view(g.shape) if g is not None else None
                j.dpa, j.dv, j.dg = dpa.data_ptr(), dv.data_ptr(), (dg.data_ptr() if dg is not None else None)
                self.dpa.append(dpa)
                _dpa_views[pa.data_ptr()] = dpa
                self.params.append(v); self.grads.append(dv if wants else None)
                if g is not None:
                    self.params.append(g); self.grads.append(dg if wants else None)
                if wants:
                    rows_bwd.extend([i] * D0)
            rows.extend([i] * D0)
            row0 += D0
            self.sig.append((v.data_ptr(), g.data_ptr() if g is not None else 0))
        self.jobs = torch.frombuffer(bytearray(bytes(jobs)), dtype=torch.uint8).to(dev)
        self.rows = torch.tensor(rows, dtype=torch.int32, device=dev)
        # the backward table re-bases row0 per job: build a second job table whose row0 counts only the rows that run
        if with_grad:
            jb = (L.PackJob * len(reqs))()
            ctypes.memmove(jb, jobs, ctypes.sizeof(jobs))
            r0 = 0
            for i, (req, ge) in enumerate(zip(reqs, geo)):
                jb[i].row0 = r0
                if req[6]:
                    r0 += ge[0]
            self.jobs_bwd = torch.frombuffer(bytearray(bytes(jb)), dtype=torch.uint8).to(dev)
            self.rows_bwd = torch.tensor(rows_bwd, dtype=torch.int32, device=dev)
        self.index = {req[0]: i for i, req in enumerate(reqs)}
        self.pa_keys = {t.data_ptr() for t in self.pa}

    def valid(self):
        """parameters still live where the job table points (they move when an optimizer re-homes them into its arena)"""
        return all((r[1].data_ptr(), r[2].data_ptr() if r[2] is not None else 0) == sg for r, sg in zip(self.reqs, self.sig))

    def run_pack(self):
        _call("evk_weight_pack_batched", _p(self.jobs), _p(self.rows), self.rows.numel())

    def run_pack_bwd(self):
        if self.rows_bwd.numel():
            _call("evk_weight_pack_bwd_batched", _p(self.jobs_bwd), _p(self.rows_bwd), self.rows_bwd.numel())

    def packed(self, i, pa=None):
        r = self.reqs[i]
        _, _, Q, D0p, D1p, _, _ = _pack_geometry(r[1], r[4], r[5])
        return PackedW(self.pa[i] if pa is None else pa, self.pb[i], D0p, D1p, Q)


class _PackAllFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, plan, *params):
        plan.arena_dpa.zero_()                     # the step's weight-gradient kernels accumulate into it
        _dpa_taken.difference_update(plan.pa_keys)
        plan.run_pack()
        ctx.plan = plan
        # FRESH tensor objects every call: returning the stored views again would hand autograd tensors that still carry
        # the previous step's history (it would chain the old graph -- recorded on another stream -- into the new one)
        return tuple(t.view(t.shape) for t in plan.pa)

    @staticmethod
    def backward(ctx, *dpas):
        plan = ctx.plan
        for d, mine in zip(dpas, plan.dpa):
            if d is not None and d.data_ptr() != mine.data_ptr():
                mine.copy_(d)                      # gradient arrived in a foreign buffer (e.g. accumulated over two uses)
        plan.run_pack_bwd()
        return (None, *plan.grads)


def pack_all(plan):
    """-> list of PackedW for every request of the plan (differentiable wrt the parameters when plan.with_grad)."""
    if plan.with_grad:
        pas = _PackAllFn.apply(plan, *plan.params)
        return [plan.packed(i, pas[i]) for i in range(len(plan.reqs))]
    with torch.no_grad():
        plan.run_pack()
    return [plan.packed(i) for i in range(len(plan.reqs))]


# ------------------------------------------------------------------------------------------------
# convolution family
# ------------------------------------------------------------------------------------------------
def _conv_out_len(Tin, Q, stride, pad, dil):
    return (Tin + 2 * pad - dil * (Q - 1) - 1) // stride + 1


def _fwd_like(x, Tin, w, ldw, w_sq, C, N, y, *, J, P, is_, off, bias=None, res=None, act=0, slope=0.0, in_len=None,
              out_len=None, G=1, drop=None, no_phase_split=0, no_grad=0):
    """one forward-like launch of the generalised conv, len(off) taps, output rows j < J; evk_gconv_fwd picks the kernel.
    Grouped convs pass G = groups (C, N are then the total channel counts).  drop = (p, stream id): dropout after the
    activation (ReLU only).  no_grad: no gradient is taken through the launch, so the library may serve it exactly."""
    B = x.shape[0]
    _, _, ldx = _rows(x)
    _, _, ldy = _rows(y)
    ldr = _rows(res)[2] if res is not None else 0
    d = _desc(x=x, w=w, y=y, res=res, bias=bias, in_len=in_len, out_len=out_len, x_sb=Tin * P * ldx, w_sq=w_sq, y_sb=J * P * ldy,
              r_sb=J * P * ldr, ldx=ldx, ldw=ldw, ldy=ldy, ldr=ldr, Z=B, G=G, C=C, N=N, Q=len(off), Tin=Tin, J=J, P=P, is_=is_,
              os_=1, Tout=J, act=act, slope=float(slope), off=off, no_phase_split=no_phase_split, no_grad=no_grad)
    if drop is not None:
        d.drop_rng, d.drop_sid, d.drop_p = rng_state(x.device).data_ptr(), int(drop[1]), float(drop[0])
    _run_desc("evk_gconv_fwd", d)


def _conv_forward(x, pa, bias, res, cfg):
    """the launch of _ConvFn's forward for a channels-last x: -> y"""
    Q, stride, pad, dil, P, G, act, slope, in_len, out_len, drop, no_grad = cfg
    B, R, C = x.shape
    assert R % P == 0
    Tin = R // P
    N, lda = pa.shape[1], pa.shape[2]
    J = _conv_out_len(Tin, Q, stride, pad, dil)
    y = torch.empty((B, J * P, N), device=x.device, dtype=torch.float32)
    if res is not None:
        res = _cl(res)
    _fwd_like(x, Tin, pa, lda, N * lda, C, N, y, J=J, P=P, is_=stride, off=[q * dil - pad for q in range(Q)], bias=bias,
              res=res, act=act, slope=slope, in_len=in_len, out_len=out_len, drop=drop, G=G, no_grad=no_grad)
    return y


class _ConvFn(torch.autograd.Function):
    """y = act(conv(x, W) + bias + res) * mask ; W packed (pa = [Q][N][C/G], pb = [Q][C/G][N])."""

    @staticmethod
    def forward(ctx, x, pa, pb, bias, res, cfg):
        x = _cl(x)
        y = _conv_forward(x, pa, bias, res, cfg)
        P, act = cfg[4], cfg[6]
        ctx.cfg = cfg
        ctx.dims = (x.shape[0], x.shape[1] // P, x.shape[2], pa.shape[1], y.shape[1] // P, pa.shape[2])
        ctx.has = (bias is not None, res is not None)
        ctx.save_for_backward(x, pa, pb, y if act else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        Q, stride, pad, dil, P, G, act, slope, in_len, out_len, drop, _ = ctx.cfg
        # dropout after a ReLU: the saved output is zero exactly where the element was dropped or the ReLU was off, so
        # the activation backward only needs the extra 1/(1-p) factor -- no mask is regenerated
        gscale = 1.0 / (1.0 - drop[0]) if drop is not None else 1.0
        B, Tin, C, N, J, lda = ctx.dims
        x, pa, pb, y = ctx.saved_tensors
        has_bias, has_res = ctx.has
        dy = dy.contiguous()
        Ro = J * P
        offs = [q * dil - pad for q in range(Q)]
        _, _, ldx = _rows(x)
        dw = _desc(x=x, y=dy, in_len=in_len, x_sb=Tin * P * ldx, w_sq=N * lda, y_sb=J * P * N, ldx=ldx, ldw=lda, ldy=N, Z=B, G=G,
                   C=C, N=N, Q=Q, Tin=Tin, J=J, P=P, is_=stride, os_=1, Tout=J, off=offs)
        tma_w = bool(ctx.needs_input_grad[1] and _lib().evk_gconv_wgrad_takes_dyt(ctypes.byref(dw)))
        want_b = has_bias and ctx.needs_input_grad[3]
        dyt = dbias = None
        if act or out_len is not None or tma_w or want_b:
            # one pass: activation backward + length mask (-> dpre), the transposed copy the TMA weight gradient reads, bias sums
            need_pre = bool(act) or out_len is not None
            dpre = torch.empty_like(dy) if need_pre else None
            ldo = (Ro + 31) // 32 * 32                                       # 128-byte aligned rows for the TMA boxes
            dyt = torch.empty((B, N, ldo), device=dy.device, dtype=torch.float32) if tma_w else None
            dw.dyt, dw.ld_dyt = _p(dyt), ldo
            dbias = _zpool.take(N, dy.device) if want_b else None
            _call("evk_dy_prep", _p(dy), N, _p(y), N, act, ctypes.c_float(slope), ctypes.c_float(gscale), _p(out_len), P, _p(dpre), N, _p(dyt),
                  ldo, N * ldo, _p(dbias), B, Ro, N)
            if need_pre:
                dy = dpre
        dx = dpa = dres = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((B, Tin * P, C), device=dy.device, dtype=torch.float32)
            d = _desc(x=dx, w=pa, y=dy, in_len=in_len, x_sb=Tin * P * C, w_sq=N * lda, y_sb=J * P * N, ldx=C, ldw=lda, ldy=N, Z=B,
                      C=C, N=N, Q=Q, G=G, Tin=Tin, J=J, P=P, is_=stride, os_=1, Tout=J, off=offs)
            if pb is not None and pb.numel():
                assert pb.shape[1] == C // G, "PB must be [Q][C/G][ldb]"
                d.wt, d.ld_wt = _p(pb), pb.shape[2]
            _run_desc("evk_gconv_dgrad", d)
        if ctx.needs_input_grad[1]:
            dpa = dpa_buffer(pa)
            dw.w, dw.y = dpa.data_ptr(), dy.data_ptr()
            _run_desc("evk_gconv_wgrad", dw)
        if has_res and ctx.needs_input_grad[4]:
            dres = dy
        return dx, dpa, None, dbias, dres, None


def conv(x, w: PackedW, bias=None, *, stride=1, pad=0, dil=1, P=1, groups=1, act=ACT_NONE, slope=0.0, res=None,
         in_len=None, out_len=None):
    """Conv1d (P == 1) / Conv2d with (k,1) kernels over a period-folded view (P == period)."""
    cfg = (w.Q, stride, pad, dil, P, groups, act, slope, in_len, out_len, None, 0)
    return _ConvFn.apply(x, w.pa, w.pb, bias, res, cfg)


def linear_rows(x, w: PackedW, bias=None, act=ACT_NONE, slope=0.0):
    """Exact-fp32 Linear of the batched token step: [..., C] with 1..64 rows in total -> [..., N], one pass over the packed
    weight (evk_gemv_rows).  A row's result does not depend on how many rows share the launch.  No gradient."""
    C = x.shape[-1]
    x2 = x.reshape(-1, C)
    if x2.stride(1) != 1:
        x2 = x2.contiguous()
    rows, N = x2.shape[0], w.pa.shape[1]
    assert w.Q == 1 and 1 <= rows <= 64 and act in (ACT_NONE, ACT_RELU, ACT_LRELU), (rows, act)
    y = torch.empty(x.shape[:-1] + (N,), device=x.device, dtype=torch.float32)
    _call_f("evk_gemv_rows", 2.0 * rows * N * C, _p(x2), x2.stride(0), rows, _p(w.pa), w.pa.shape[2], _p(bias), _p(y), N, N, C,
            int(act), ctypes.c_float(float(slope)))
    return y


def linear(x, w: PackedW, bias=None, act=ACT_NONE, slope=0.0, out_len=None, in_len=None, res=None, drop=None):
    """nn.Linear / 1x1 conv on [B, T, C] or [rows, C].  drop = (p, tag): dropout_p(relu(x W^T + b)), act must be ReLU.
    Without autograd recording, the library may serve a launch of a few rows exactly in fp32 (evk_gconv_fwd's route 0)."""
    if drop is not None and drop[0] > 0.0:
        assert act == ACT_RELU, "linear(drop=...) needs act=ACT_RELU: the backward recovers the mask from the saved output"
        drop = (float(drop[0]), stream_id(drop[1]))
    else:
        drop = None
    no_grad = int(not torch.is_grad_enabled())
    flat = x.dim() == 2
    if flat:
        x, res, in_len, out_len = x.unsqueeze(0), res.unsqueeze(0) if res is not None else None, None, None
    cfg = (w.Q, 1, 0, 1, 1, 1, act, slope, in_len, out_len, drop, no_grad)
    # no autograd recording: the launch alone, without the Function's bookkeeping (host time of the skinny decode Linears)
    y = _conv_forward(_cl(x), w.pa, bias, res, cfg) if no_grad else _ConvFn.apply(x, w.pa, w.pb, bias, res, cfg)
    return y.squeeze(0) if flat else y


class _ConvTFn(torch.autograd.Function):
    """ConvTranspose1d: v [Cin][Cout][Q] packed as pa = [Q][Cin][Cout], pb = [Q][Cout][Cin].  It is the conv with Cout
    input and Cin output channels, weight PA, run backwards: the forward is that conv's data gradient, the data gradient
    its forward."""

    @staticmethod
    def forward(ctx, x, pa, pb, bias, cfg, out_len=None):
        Q, stride, pad = cfg
        x = _cl(x)
        B, Tin, Cin = x.shape
        Cout, lda = pb.shape[1], pa.shape[2]
        Tout = (Tin - 1) * stride - 2 * pad + Q
        y = torch.empty((B, Tout, Cout), device=x.device, dtype=torch.float32)
        _, _, ldx = _rows(x)
        d = _desc(x=y, w=pa, y=x, bias=bias, out_len=out_len, x_sb=Tout * Cout, w_sq=Cin * lda, y_sb=Tin * ldx, ldx=Cout, ldw=lda, ldy=ldx, Z=B,
                  C=Cout, N=Cin, Q=Q, Tin=Tout, J=Tin, P=1, is_=stride, os_=1, Tout=Tin, off=[q - pad for q in range(Q)])
        d.wt, d.ld_wt = _p(pb), pb.shape[2]
        _run_desc("evk_gconv_dgrad", d)
        ctx.cfg = cfg
        ctx.dims = (B, Tin, Cin, Cout, Tout)
        ctx.save_for_backward(x, pa)
        return y

    @staticmethod
    def backward(ctx, dy):
        Q, stride, pad = ctx.cfg
        B, Tin, Cin, Cout, Tout = ctx.dims
        x, pa = ctx.saved_tensors
        dy = dy.contiguous()
        lda = pa.shape[2]
        off = [q - pad for q in range(Q)]
        dx = dpa = dbias = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((B, Tin, Cin), device=dy.device, dtype=torch.float32)
            _fwd_like(dy, Tout, pa, lda, Cin * lda, Cout, Cin, dx, J=Tin, P=1, is_=stride, off=off, no_phase_split=1)
        if ctx.needs_input_grad[1]:
            dpa = dpa_buffer(pa)
            _, _, ldx = _rows(x)
            # dPA[q][ci][co] += sum_t X[t][ci] * dY[t*stride - pad + q][co]: "x" role = dY (shifted), "y" role = X
            d = _desc(x=dy, w=dpa, y=x, x_sb=Tout * Cout, w_sq=Cin * lda, y_sb=Tin * ldx, ldx=Cout, ldw=lda, ldy=ldx, Z=B,
                      C=Cout, N=Cin, Q=Q, Tin=Tout, J=Tin, P=1, is_=stride, os_=1, Tout=Tin, off=off)
            _run_desc("evk_gconv_wgrad", d)
        if ctx.needs_input_grad[3]:
            dbias = torch.empty(Cout, device=dy.device, dtype=torch.float32)
            _call("evk_colsum", _p(dy), B * Tout, Cout, Cout, _p(dbias), 0)
        return dx, dpa, None, dbias, None, None


def conv_transpose(x, w: PackedW, bias, *, stride, pad, out_len=None):
    """ConvTranspose1d.  out_len (inference, int32 device [B]): output rows past out_len[b] are written as zero; x's rows past
    a row's input length must be zero (evk_gconv_dgrad)."""
    assert out_len is None or not torch.is_grad_enabled(), "conv_transpose(out_len=...) has no backward"
    return _ConvTFn.apply(x, w.pa, w.pb, bias, (w.Q, stride, pad), out_len)


# ------------------------------------------------------------------------------------------------
# element-wise family
# ------------------------------------------------------------------------------------------------
class _UnaryFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, op, alpha):
        x = _cl(x)
        rows, C, ld = _rows(x)
        y = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        _call("evk_unary", op, ctypes.c_float(alpha), _p(x), ld, _p(y), C, rows, C)
        ctx.save_for_backward(x)
        ctx.op, ctx.alpha = op, alpha
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        rows, C, ld = _rows(x)
        dy = dy.contiguous()
        dx = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        _call("evk_unary_bwd", ctx.op, ctypes.c_float(ctx.alpha), _p(x), ld, _p(dy), C, _p(dx), C, rows, C)
        return dx, None, None


def lrelu(x, slope):
    return _UnaryFn.apply(x, UN_LRELU, slope)


def tanh(x):
    return _UnaryFn.apply(x, UN_TANH, 0.0)


def mish(x):
    return _UnaryFn.apply(x, UN_MISH, 0.0)


def scale(x, alpha):
    return _UnaryFn.apply(x, UN_SCALE, alpha)


def gelu(x):
    """exact (erf) GELU, inference only (HuBERT): no gradient."""
    x = _cl(x.detach())
    rows, C, ld = _rows(x)
    y = torch.empty(x.shape, device=x.device, dtype=torch.float32)
    _call("evk_unary", UN_GELU, ctypes.c_float(0.0), _p(x), ld, _p(y), C, rows, C)
    return y


def instnorm_cl(x, gamma, beta, eps=1e-5, gelu_after=False, lens=None):
    """GroupNorm(C, C) over time of a channels-last [B, T, C] tensor (+ optional exact GELU); inference only.  lens (int32
    device [B], optional): item b is normalised over its first lens[b] frames and the frames after them are 0."""
    x = _cl(x.detach())
    B, T, C = x.shape
    _, _, ld = _rows(x)
    assert lens is None or (lens.dtype == torch.int32 and lens.is_cuda and lens.numel() == B)
    y = torch.empty((B, T, C), device=x.device, dtype=torch.float32)
    _call("evk_instnorm_cl", _p(x), ld, _p(gamma.detach().contiguous()), _p(beta.detach().contiguous()), ctypes.c_float(eps),
          1 if gelu_after else 0, _p(y), C, B, T, C, _p(None if lens is None else lens.contiguous()))
    return y


def _axpby_raw(a, alpha, b=None, beta=0.0, c=None, gamma=0.0, length=None, T=0):
    a = _cl(a)
    rows, C, lda = _rows(a)
    y = torch.empty(a.shape, device=a.device, dtype=torch.float32)
    ldb = ldc = 0
    if b is not None:
        b = _cl(b)
        ldb = _rows(b)[2]
    if c is not None:
        c = _cl(c)
        ldc = _rows(c)[2]
    _call("evk_axpby", _p(a), lda, ctypes.c_float(alpha), _p(b), ldb, ctypes.c_float(beta), _p(c), ldc,
          ctypes.c_float(gamma), _p(y), C, rows, C, _p(length), T)
    return y


class _AxpbyFn(torch.autograd.Function):
    """y = mask(alpha*a + beta*b + gamma*c)"""

    @staticmethod
    def forward(ctx, a, b, c, alpha, beta, gamma, length):
        T = a.shape[1] if a.dim() == 3 else 0
        ctx.k = (alpha, beta, gamma, length, T)
        return _axpby_raw(a, alpha, b, beta, c, gamma, length, T)

    @staticmethod
    def backward(ctx, dy):
        alpha, beta, gamma, length, T = ctx.k
        need = ctx.needs_input_grad
        if length is None and alpha == 1.0 and beta == 1.0 and gamma in (0.0, 1.0):
            return (dy if need[0] else None, dy if need[1] else None, dy if need[2] else None, None, None, None, None)
        dy = dy.contiguous()
        base = _axpby_raw(dy, 1.0, length=length, T=T) if length is not None else dy
        outs = []
        for k, coef in enumerate((alpha, beta, gamma)):
            if not need[k]:
                outs.append(None)
            elif coef == 1.0:
                outs.append(base)
            else:
                outs.append(_axpby_raw(base, coef))
        return (*outs, None, None, None, None)


def add(a, b, alpha=1.0, beta=1.0, length=None):
    return _AxpbyFn.apply(a, b, None, alpha, beta, 0.0, length)


def add3(a, b, c, alpha=1.0, beta=1.0, gamma=1.0):
    return _AxpbyFn.apply(a, b, c, alpha, beta, gamma, None)


def rowmask(x, length):
    return _AxpbyFn.apply(x, None, None, 1.0, 0.0, 0.0, length)


class _AddBvecFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, v):
        x = _cl(x)
        B, T, C = x.shape
        _, _, ldx = _rows(x)
        v2 = v.reshape(B, C).contiguous()
        y = torch.empty((B, T, C), device=x.device, dtype=torch.float32)
        _call("evk_add_bvec", _p(x), ldx, _p(v2), C, _p(y), C, B, T, C)
        ctx.dims = (B, T, C, tuple(v.shape))
        return y

    @staticmethod
    def backward(ctx, dy):
        B, T, C, vshape = ctx.dims
        dv = None
        if ctx.needs_input_grad[1]:
            dy = dy.contiguous()
            dv = torch.empty((B, C), device=dy.device, dtype=torch.float32)
            _call("evk_masked_mean", _p(dy), C, _p(dv), C, B, T, C, None, 0)
            dv = _axpby_raw(dv, float(T)).reshape(vshape)
        return dy, dv


def add_bvec(x, v):
    """x [B,T,C] + v [B,1,C] (broadcast over time)."""
    return _AddBvecFn.apply(x, v)


class _WnGateFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, g):
        a = _cl(a)
        B, T, H2 = a.shape
        H = H2 // 2
        _, _, lda = _rows(a)
        ldg = 0
        if g is not None:
            g = _cl(g)
            ldg = _rows(g)[2]
        y = torch.empty((B, T, H), device=a.device, dtype=torch.float32)
        _call("evk_wn_gate", _p(a), lda, _p(g), ldg, _p(y), H, B, T, H)
        ctx.save_for_backward(a, g)
        return y

    @staticmethod
    def backward(ctx, dy):
        a, g = ctx.saved_tensors
        B, T, H2 = a.shape
        H = H2 // 2
        _, _, lda = _rows(a)
        ldg = _rows(g)[2] if g is not None else 0
        dy = dy.contiguous()
        da = torch.empty((B, T, H2), device=a.device, dtype=torch.float32)
        _call("evk_wn_gate_bwd", _p(a), lda, _p(g), ldg, _p(dy), H, _p(da), H2, B, T, H)
        dg = None
        if g is not None and ctx.needs_input_grad[1]:
            dg = torch.empty((B, H2), device=a.device, dtype=torch.float32)
            _call("evk_masked_mean", _p(da), H2, _p(dg), H2, B, T, H2, None, 0)
            dg = _axpby_raw(dg, float(T)).reshape(g.shape)
        return da, dg


def wn_gate(a, g):
    """tanh(a[..., :H] + g[..., :H]) * sigmoid(a[..., H:] + g[..., H:]); g is [B, 1, 2H] (broadcast over time)."""
    return _WnGateFn.apply(a, g)


class _GluResFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, h):
        h = _cl(h)
        rows, C2, ldh = _rows(h)
        C = C2 // 2
        ldx = 0
        if x is not None:
            x = _cl(x)
            ldx = _rows(x)[2]
        y = torch.empty((*h.shape[:-1], C), device=h.device, dtype=torch.float32)
        _call("evk_glu_res", _p(x), ldx, _p(h), ldh, _p(y), C, rows, C)
        ctx.save_for_backward(h)
        ctx.has_x = x is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        (h,) = ctx.saved_tensors
        rows, C2, ldh = _rows(h)
        C = C2 // 2
        dy = dy.contiguous()
        dh = torch.empty(h.shape, device=h.device, dtype=torch.float32)
        _call("evk_glu_res_bwd", _p(h), ldh, _p(dy), C, _p(dh), C2, rows, C)
        return (dy if ctx.has_x else None), dh


def glu_res(x, h):
    """x + h[..., :C] * sigmoid(h[..., C:])   (x may be None)."""
    return _GluResFn.apply(x, h)


class _CatFlipFn(torch.autograd.Function):
    """flip_channels(cat([x0, x1], -1)) -- the coupling layer's cat + Flip (modules.py:376-383,452-454) in one pass."""

    @staticmethod
    def forward(ctx, x0, x1):
        x0, x1 = _cl(x0), _cl(x1)
        rows, C0, ld0 = _rows(x0)
        _, C1, ld1 = _rows(x1)
        y = torch.empty((*x0.shape[:-1], C0 + C1), device=x0.device, dtype=torch.float32)
        _call("evk_flip_channels", _p(x1), ld1, _p(y), C0 + C1, rows, C1)
        _call("evk_flip_channels", _p(x0), ld0, _p(y[..., C1:]), C0 + C1, rows, C0)
        ctx.k = (C0, C1)
        return y

    @staticmethod
    def backward(ctx, dy):
        C0, C1 = ctx.k
        dy = dy.contiguous()
        rows = dy.numel() // (C0 + C1)
        d0 = torch.empty((*dy.shape[:-1], C0), device=dy.device, dtype=torch.float32)
        d1 = torch.empty((*dy.shape[:-1], C1), device=dy.device, dtype=torch.float32)
        _call("evk_flip_channels", _p(dy), C0 + C1, _p(d1), C1, rows, C1)
        _call("evk_flip_channels", _p(dy[..., C1:]), C0 + C1, _p(d0), C0, rows, C0)
        return d0, d1


def cat_flip(x0, x1):
    return _CatFlipFn.apply(x0, x1)


class _CatBatchFn(torch.autograd.Function):
    """cat([a, b], dim=0) with a copy kernel (discriminators run real and generated audio as one 2B batch)."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        y = torch.empty((a.shape[0] + b.shape[0], *a.shape[1:]), device=a.device, dtype=torch.float32)
        na, nb = a.numel(), b.numel()
        one, zero = ctypes.c_float(1.0), ctypes.c_float(0.0)
        _call("evk_axpby", _p(a), na, one, None, 0, zero, None, 0, zero, _p(y), na, 1, na, None, 0)
        _call("evk_axpby", _p(b), nb, one, None, 0, zero, None, 0, zero, _p(y[a.shape[0]:]), nb, 1, nb, None, 0)
        ctx.na = a.shape[0]
        return y

    @staticmethod
    def backward(ctx, dy):
        na = ctx.na
        return (dy[:na] if ctx.needs_input_grad[0] else None), (dy[na:] if ctx.needs_input_grad[1] else None)


def cat_batch(a, b):
    return _CatBatchFn.apply(a, b)


class _PadChFn(torch.autograd.Function):
    """[.., C] -> [.., Cp] zero-padded channels (1-channel waveforms are padded to 4 so that the first discriminator
    layers run on the 16-byte-tiled tensor-core kernels)."""

    @staticmethod
    def forward(ctx, x, Cp):
        x = _cl(x)
        rows, C, ld = _rows(x)
        y = torch.zeros((*x.shape[:-1], Cp), device=x.device, dtype=torch.float32)
        _call("evk_axpby", _p(x), ld, ctypes.c_float(1.0), None, 0, ctypes.c_float(0.0), None, 0, ctypes.c_float(0.0), _p(y),
              Cp, rows, C, None, 0)
        ctx.k = (C, Cp)
        return y

    @staticmethod
    def backward(ctx, dy):
        C, Cp = ctx.k
        dy = dy.contiguous()
        rows = dy.numel() // Cp
        dx = torch.empty((*dy.shape[:-1], C), device=dy.device, dtype=torch.float32)
        _call("evk_axpby", _p(dy), Cp, ctypes.c_float(1.0), None, 0, ctypes.c_float(0.0), None, 0, ctypes.c_float(0.0),
              _p(dx), C, rows, C, None, 0)
        return dx, None


def pad_channels(x, Cp):
    return x if x.shape[-1] >= Cp else _PadChFn.apply(x, Cp)


class _TakeChFn(torch.autograd.Function):
    """contiguous copy of the first C channels (inverse of pad_channels)."""

    @staticmethod
    def forward(ctx, x, C):
        x = _cl(x)
        rows, Cp, ld = _rows(x)
        y = torch.empty((*x.shape[:-1], C), device=x.device, dtype=torch.float32)
        _call("evk_axpby", _p(x), ld, ctypes.c_float(1.0), None, 0, ctypes.c_float(0.0), None, 0, ctypes.c_float(0.0), _p(y),
              C, rows, C, None, 0)
        ctx.k = (C, Cp)
        return y

    @staticmethod
    def backward(ctx, dy):
        C, Cp = ctx.k
        dy = dy.contiguous()
        rows = dy.numel() // C
        dx = torch.zeros((*dy.shape[:-1], Cp), device=dy.device, dtype=torch.float32)
        _call("evk_axpby", _p(dy), C, ctypes.c_float(1.0), None, 0, ctypes.c_float(0.0), None, 0, ctypes.c_float(0.0),
              _p(dx), Cp, rows, C, None, 0)
        return dx, None


def take_channels(x, C):
    return x if x.shape[-1] == C else _TakeChFn.apply(x, C)


class _ReparamFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, stats, noise, length):
        stats, noise = _cl(stats), _cl(noise)
        B, T, C2 = stats.shape
        C = C2 // 2
        z = torch.empty((B, T, C), device=stats.device, dtype=torch.float32)
        _call("evk_reparam", _p(stats), _rows(stats)[2], _p(noise), _rows(noise)[2], _p(z), C, B, T, C, _p(length))
        ctx.save_for_backward(stats, noise)
        ctx.length = length
        return z

    @staticmethod
    def backward(ctx, dz):
        stats, noise = ctx.saved_tensors
        B, T, C2 = stats.shape
        C = C2 // 2
        dz = dz.contiguous()
        ds = torch.empty((B, T, C2), device=stats.device, dtype=torch.float32)
        _call("evk_reparam_bwd", _p(stats), _rows(stats)[2], _p(noise), _rows(noise)[2], _p(dz), C, _p(ds), C2, B, T, C,
              _p(ctx.length))
        return ds, None, None


def reparam(stats, noise, length):
    """z = (m + noise * exp(logs)) * mask with stats = [m | logs]."""
    return _ReparamFn.apply(stats, noise, length)


class _FlipFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _cl(x)
        rows, C, ld = _rows(x)
        y = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        _call("evk_flip_channels", _p(x), ld, _p(y), C, rows, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        rows, C, ld = _rows(dy)
        dx = torch.empty_like(dy)
        _call("evk_flip_channels", _p(dy), ld, _p(dx), C, rows, C)
        return dx


def flip_channels(x):
    return _FlipFn.apply(x)


class _SliceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ids, mul, seg):
        x = _cl(x)
        B, T, C = x.shape
        _, _, ld = _rows(x)
        y = torch.empty((B, seg, C), device=x.device, dtype=torch.float32)
        _call("evk_slice_rows", _p(x), ld, T, _p(ids), mul, _p(y), C, B, seg, C, 0)
        ctx.k = (ids, mul, seg, B, T, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        ids, mul, seg, B, T, C = ctx.k
        dy = dy.contiguous()
        dx = torch.zeros((B, T, C), device=dy.device, dtype=torch.float32)
        _call("evk_slice_rows", _p(dx), C, T, _p(ids), mul, _p(dy), C, B, seg, C, 1)
        return dx, None, None, None


def slice_rows(x, ids, seg, mul=1):
    """commons.slice_segments on a channels-last tensor; ids int64 device [B]."""
    return _SliceFn.apply(x, ids, mul, seg)


class _ReflectPadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, Tp):
        x = x.contiguous()
        B, T, _ = x.shape
        y = torch.empty((B, Tp, 1), device=x.device, dtype=torch.float32)
        _call("evk_reflect_pad_right", _p(x), T, _p(y), Tp, B, 0)
        ctx.k = (B, T, Tp)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, T, Tp = ctx.k
        dy = dy.contiguous()
        dx = torch.empty((B, T, 1), device=dy.device, dtype=torch.float32)
        _call("evk_reflect_pad_right", _p(dx), T, _p(dy), Tp, B, 1)
        return dx, None


def reflect_pad_right(x, Tp):
    return x if Tp == x.shape[1] else _ReflectPadFn.apply(x, Tp)


def widen_to_pitch(x):
    """[B, T, C] view whose row pitch is wider than C (|X| from mel_frontend, to_channels_last(pad_to=4)) -> the [B, T, pitch]
    view over the same memory.  The producers zero the pitch columns, so the wide view is a valid 16-byte tileable operand."""
    if x.dim() != 3 or x.stride(2) != 1 or x.stride(1) == x.shape[2]:
        return x
    ld = x.stride(1)
    assert ld > x.shape[2] and ld % 4 == 0 and x.stride(0) == x.shape[1] * ld
    return torch.as_strided(x, (x.shape[0], x.shape[1], ld), x.stride(), x.storage_offset())


def to_channels_last(x, pad_to=None):
    """[B, C, T] -> [B, T, C] (new memory; pitch rounded up to `pad_to` channels, returned as a view)."""
    x = x.contiguous()
    B, C, T = x.shape
    ld = C if pad_to is None else (C + pad_to - 1) // pad_to * pad_to
    buf = (torch.zeros if ld != C else torch.empty)((B, T, ld), device=x.device, dtype=torch.float32)   # pitch columns stay zero
    _call("evk_transpose_bct_btc", _p(x), _p(buf), B, C, T, ld, 1)
    return buf[:, :, :C] if ld != C else buf


def to_channels_first(x):
    """[B, T, C] -> [B, C, T]"""
    x = _cl(x)
    B, T, C = x.shape
    _, _, ld = _rows(x)
    y = torch.empty((B, C, T), device=x.device, dtype=torch.float32)
    _call("evk_transpose_bct_btc", _p(x), _p(y), B, C, T, ld, 0)
    return y


class _EmbFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, idx, rep):
        table = table.contiguous()
        rows = idx.numel() * rep
        C = table.shape[1]
        y = torch.empty((*idx.shape[:-1], idx.shape[-1] * rep, C), device=table.device, dtype=torch.float32)
        idx = idx.contiguous()
        _call("evk_embedding", _p(table), C, _p(idx), rows, rep, _p(y), C, C)
        ctx.save_for_backward(idx)
        ctx.k = (tuple(table.shape), rep)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        shape, rep = ctx.k
        assert rep == 1
        dy = dy.contiguous()
        dt = torch.zeros(shape, device=dy.device, dtype=torch.float32)
        _call("evk_embedding_bwd", _p(dy), shape[1], _p(idx), idx.numel(), _p(dt), shape[1], shape[1], shape[0])
        return dt, None, None


def embedding(table, idx, rep=1):
    """idx int64 [B, T] -> [B, T*rep, C] (rep = nearest-neighbour upsample factor along time)."""
    return _EmbFn.apply(table, idx, rep)


class _MaskedMeanFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, length):
        x = _cl(x)
        B, T, C = x.shape
        y = torch.empty((B, C), device=x.device, dtype=torch.float32)
        _call("evk_masked_mean", _p(x), _rows(x)[2], _p(y), C, B, T, C, _p(length), 0)
        ctx.k = (B, T, C, length)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, T, C, length = ctx.k
        dy = dy.contiguous()
        dx = torch.empty((B, T, C), device=dy.device, dtype=torch.float32)
        _call("evk_masked_mean", _p(dx), C, _p(dy), C, B, T, C, _p(length), 1)
        return dx, None


def masked_mean(x, length):
    return _MaskedMeanFn.apply(x, length)


class _DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p, sid):
        x = x.contiguous()
        y = torch.empty_like(x)
        _call("evk_dropout", _p(x), _p(y), x.numel(), ctypes.c_float(p), _p(rng_state(x.device)), ctypes.c_uint64(sid))
        ctx.k = (p, sid)
        return y

    @staticmethod
    def backward(ctx, dy):
        p, sid = ctx.k
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        _call("evk_dropout", _p(dy), _p(dx), dy.numel(), ctypes.c_float(p), _p(rng_state(dy.device)), ctypes.c_uint64(sid))
        return dx, None, None


def dropout(x, p, tag):
    """inverted dropout; the mask is regenerated (not stored) in backward from (seed, offset, stream id)."""
    if p <= 0.0:
        return x
    return _DropoutFn.apply(x, p, stream_id(tag))


def randn(shape, tag, device=None, state=None):
    """standard normal draws keyed by the library's RNG state, or by `state` (int64 device [2] = (seed, offset)) when given"""
    y = torch.empty(shape, device=device or "cuda", dtype=torch.float32)
    _call("evk_randn", _p(y), y.numel(), _p(rng_state(y.device) if state is None else state), ctypes.c_uint64(stream_id(tag)))
    return y


def rand_slice_ids(length, seg, tag="slice"):
    ids = torch.empty(length.shape[0], device=length.device, dtype=torch.int64)
    _call("evk_rand_slice_ids", _p(ids), _p(length), length.shape[0], seg, _p(rng_state(length.device)),
          ctypes.c_uint64(stream_id(tag)))
    return ids


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps):
        x = _cl(x)
        rows, C, ldx = _rows(x)
        ldr = 0
        if res is not None:
            res = _cl(res)
            ldr = _rows(res)[2]
        y = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        stats = torch.empty((rows, 2), device=x.device, dtype=torch.float32)
        _call("evk_layernorm_fwd", _p(x), ldx, _p(res), ldr, _p(gamma), _p(beta), ctypes.c_float(eps), _p(y), C, _p(stats),
              rows, C)
        ctx.save_for_backward(x, res, gamma, stats)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, res, gamma, stats = ctx.saved_tensors
        rows, C, ldx = _rows(x)
        ldr = _rows(res)[2] if res is not None else 0
        dy = dy.contiguous()
        dx = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        dgb = torch.zeros((2, C), device=x.device, dtype=torch.float32)
        _call("evk_layernorm_bwd", _p(x), ldx, _p(res), ldr, _p(gamma), _p(stats), _p(dy), C, _p(dx), C, _p(dgb[0]),
              _p(dgb[1]), rows, C)
        return dx, (dx if res is not None else None), dgb[0], dgb[1], None


class _LayerNormDropFn(torch.autograd.Function):
    """LayerNorm(x + dropout_p(res)) in one kernel; the backward regenerates the mask and emits dres = dx * mask / (1-p)."""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps, p, sid):
        x, res = x.contiguous(), res.contiguous()
        C = x.shape[-1]
        rows = x.numel() // C
        y = torch.empty_like(x)
        stats = torch.empty((rows, 2), device=x.device, dtype=torch.float32)
        gamma, beta = gamma.contiguous(), beta.contiguous()
        _call("evk_layernorm_drop_fwd", _p(x), _p(res), _p(gamma), _p(beta), ctypes.c_float(eps), ctypes.c_float(p), _p(rng_state(x.device)),
              ctypes.c_uint64(sid), _p(y), _p(stats), rows, C)
        ctx.save_for_backward(x, res, gamma, stats)
        ctx.k = (p, sid, rows, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, res, gamma, stats = ctx.saved_tensors
        p, sid, rows, C = ctx.k
        dy = dy.contiguous()
        if dy.data_ptr() % 16:
            dy = dy.clone()
        dx, dres = torch.empty_like(x), torch.empty_like(x)
        dgb = torch.zeros((2, C), device=x.device, dtype=torch.float32)
        _call("evk_layernorm_drop_bwd", _p(x), _p(res), _p(gamma), _p(stats), _p(dy), ctypes.c_float(p), _p(rng_state(x.device)),
              ctypes.c_uint64(sid), _p(dx), _p(dres), _p(dgb[0]), _p(dgb[1]), rows, C)
        return dx, dres, dgb[0], dgb[1], None, None, None


def layernorm(x, gamma, beta, res=None, eps=1e-5, res_drop=None):
    """LayerNorm over channels of (x + res).  res_drop = (p, tag): LayerNorm(x + dropout_p(res)) with the dropout fused into the
    kernel (C % 4 == 0, C <= 512, contiguous tensors); other shapes apply the dropout as a separate kernel."""
    if res_drop is not None and res_drop[0] > 0.0 and res is not None:
        C = x.shape[-1]
        if C % 4 == 0 and C <= 512 and x.data_ptr() % 16 == 0 and res.data_ptr() % 16 == 0 and x.is_contiguous() and res.is_contiguous():
            return _LayerNormDropFn.apply(x, res, gamma, beta, eps, float(res_drop[0]), stream_id(res_drop[1]))
        res = dropout(res, res_drop[0], res_drop[1])
    return _LayerNormFn.apply(x, res, gamma, beta, eps)


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _transpose_cl(x, ldT):
    """[B, T, C] -> [B, C, ldT] (time-contiguous copy used as the K-major operand of P.V and dS.K)."""
    x = _cl(x)
    B, T, C = x.shape
    _, _, ld = _rows(x)
    y = torch.empty((B, C, ldT), device=x.device, dtype=torch.float32)
    # evk_transpose (to_btc=0) reads [B][T][ld] and writes [B][C][T]; write with row pitch ldT via per-batch view
    if ldT == T:
        _call("evk_transpose_bct_btc", _p(x), _p(y), B, C, T, ld, 0)
    else:
        tmp = torch.empty((B, C, T), device=x.device, dtype=torch.float32)
        _call("evk_transpose_bct_btc", _p(x), _p(tmp), B, C, T, ld, 0)
        y.zero_()
        _call("evk_axpby", _p(tmp), T, ctypes.c_float(1.0), None, 0, ctypes.c_float(0.0), None, 0, ctypes.c_float(0.0),
              _p(y), ldT, B * C, T, None, 0)
    return y


def _bgemm(fn, x, x_sb, x_sh, ldx, w, w_sb, w_sh, ldw, y, y_sb, y_sh, ldy, Z, H, C, N, rows):
    d = _desc(x=x, w=w, y=y, x_sb=x_sb, x_sh=x_sh, w_sb=w_sb, w_sh=w_sh, y_sb=y_sb, y_sh=y_sh, ldx=ldx, ldw=ldw, ldy=ldy,
              Z=Z, H=H, C=C, N=N, Q=1, Tin=rows, J=rows, P=1, is_=1, os_=1, Tout=rows)
    _run_desc(fn, d)


class _AttnFn(torch.autograd.Function):
    """softmax((q k^T + q Ek^T) * scale, masked) (dropout) (v + Ev band) -- attentions.py:243-292."""

    @staticmethod
    def forward(ctx, q, k, v, Ek, Ev, cfg):
        H, win, scale_, fill, qlen, klen, p_drop, sid = cfg
        q, k, v = _cl(q), _cl(k), _cl(v)
        B, Tq, C = q.shape
        Tk = k.shape[1]
        dk = C // H
        Z = B * H
        ldq, ldk, ldv = _rows(q)[2], _rows(k)[2], _rows(v)[2]
        ldS = (Tk + 3) // 4 * 4
        S = torch.empty((Z, Tq, ldS), device=q.device, dtype=torch.float32)
        # S[z][i][j] = q_i . k_j
        _bgemm("evk_gconv_fwd", q, Tq * ldq, dk, ldq, k, Tk * ldk, dk, ldk, S, H * Tq * ldS, Tq * ldS, ldS, Z, H, dk, Tk, Tq)
        rel = None
        if win is not None:
            Ekc = Ek.reshape(2 * win + 1, dk).contiguous()
            rel = torch.empty((Z, Tq, 2 * win + 1), device=q.device, dtype=torch.float32)
            _call("evk_relk_logits", _p(q), ldq, _p(Ekc), B, H, Tq, dk, win, _p(rel))
        _call("evk_attn_softmax", _p(S), ldS, Z, H, Tq, Tk, ctypes.c_float(scale_), _p(rel), win or 0, _p(qlen), _p(klen),
              ctypes.c_float(fill))
        P = S
        Pd = P
        if p_drop > 0.0:
            Pd = torch.empty_like(P)
            _call("evk_dropout", _p(P), _p(Pd), P.numel(), ctypes.c_float(p_drop), _p(rng_state(q.device)),
                  ctypes.c_uint64(sid))
        ldT = ldS
        Vt = _transpose_cl(v, ldT)                                   # [B, C, ldT]
        out = torch.empty((B, Tq, C), device=q.device, dtype=torch.float32)
        _bgemm("evk_gconv_fwd", Pd, H * Tq * ldS, Tq * ldS, ldS, Vt, C * ldT, dk * ldT, ldT, out, Tq * C, dk, C, Z, H, Tk,
               dk, Tq)
        band = None
        if win is not None:
            Evc = Ev.reshape(2 * win + 1, dk).contiguous()
            band = torch.empty((Z, Tq, 2 * win + 1), device=q.device, dtype=torch.float32)
            _call("evk_attn_band", _p(Pd), ldS, _p(band), Z, Tq, Tk, win, 1)
            _call("evk_relv_out", _p(band), _p(Evc), B, H, Tq, dk, win, _p(out), C)
        ctx.cfg = cfg
        ctx.save_for_backward(q, k, v, P, Pd if p_drop > 0.0 else None, band, Ek, Ev)
        return out

    @staticmethod
    def backward(ctx, dout):
        H, win, scale_, fill, qlen, klen, p_drop, sid = ctx.cfg
        q, k, v, P, Pd, band, Ek, Ev = ctx.saved_tensors
        if Pd is None:
            Pd = P
        B, Tq, C = q.shape
        Tk = k.shape[1]
        dk = C // H
        Z = B * H
        ldq, ldk, ldv = _rows(q)[2], _rows(k)[2], _rows(v)[2]
        ldS = P.shape[2]
        dout = dout.contiguous()
        dev = q.device
        W = 2 * win + 1 if win is not None else 0
        # dPd = dO V^T
        dP = torch.empty((Z, Tq, ldS), device=dev, dtype=torch.float32)
        _bgemm("evk_gconv_fwd", dout, Tq * C, dk, C, v, Tk * ldv, dk, ldv, dP, H * Tq * ldS, Tq * ldS, ldS, Z, H, dk, Tk, Tq)
        dEk = dEv = None
        if win is not None:
            Evc = Ev.reshape(W, dk).contiguous()
            dband = torch.empty((Z, Tq, W), device=dev, dtype=torch.float32)
            dEv = torch.zeros((W, dk), device=dev, dtype=torch.float32)
            _call("evk_relv_bwd", _p(band), _p(dout), C, _p(Evc), B, H, Tq, dk, win, _p(dband), _p(dEv))
            _call("evk_attn_band", _p(dP), ldS, _p(dband), Z, Tq, Tk, win, 0)
        # dV[b][j][h*dk+d] = sum_i Pd[z][i][j] dO[b][i][h*dk+d]
        dv = torch.zeros((B, Tk, C), device=dev, dtype=torch.float32)
        _bgemm("evk_gconv_wgrad", dout, Tq * C, dk, C, dv, Tk * C, dk, C, Pd, H * Tq * ldS, Tq * ldS, ldS, Z, H, dk, Tk, Tq)
        if p_drop > 0.0:
            dPn = torch.empty_like(dP)
            _call("evk_dropout", _p(dP), _p(dPn), dP.numel(), ctypes.c_float(p_drop), _p(rng_state(dev)), ctypes.c_uint64(sid))
            dP = dPn
        drel = torch.empty((Z, Tq, W), device=dev, dtype=torch.float32) if win is not None else None
        _call("evk_attn_softmax_bwd", _p(P), _p(dP), ldS, Z, H, Tq, Tk, ctypes.c_float(scale_), _p(drel), win or 0, _p(qlen),
              _p(klen))
        dS = dP
        # dQ = dS K  (K^T as the K-major operand)
        Kt = _transpose_cl(k, ldS)
        dq = torch.empty((B, Tq, C), device=dev, dtype=torch.float32)
        _bgemm("evk_gconv_fwd", dS, H * Tq * ldS, Tq * ldS, ldS, Kt, C * ldS, dk * ldS, ldS, dq, Tq * C, dk, C, Z, H, Tk, dk, Tq)
        # dK[b][j][h*dk+d] = sum_i dS[z][i][j] q[b][i][h*dk+d]
        dkk = torch.zeros((B, Tk, C), device=dev, dtype=torch.float32)
        _bgemm("evk_gconv_wgrad", q, Tq * ldq, dk, ldq, dkk, Tk * C, dk, C, dS, H * Tq * ldS, Tq * ldS, ldS, Z, H, dk, Tk, Tq)
        if win is not None:
            Ekc = Ek.reshape(W, dk).contiguous()
            dEk = torch.zeros((W, dk), device=dev, dtype=torch.float32)
            _call("evk_relk_bwd", _p(drel), _p(q), ldq, _p(Ekc), B, H, Tq, dk, win, _p(dq), C, _p(dEk))
            dEk = dEk.reshape(Ek.shape)
            dEv = dEv.reshape(Ev.shape)
        return dq, dkk, dv, dEk, dEv, None


def attention(q, k, v, *, heads, scale, Ek=None, Ev=None, window=None, fill=-1e4, qlen=None, klen=None, p_drop=0.0,
              tag="attn"):
    cfg = (heads, window, float(scale), float(fill), qlen, klen, float(p_drop), stream_id(tag))
    return _AttnFn.apply(q, k, v, Ek, Ev, cfg)


def attention_pad(qkv, *, heads, lens, scale):
    """Fused bidirectional attention, head dim 64, inference only (evk_attn_pad_fwd): qkv [B, L, >= 3*heads*64] holds q | k | v
    column blocks (one packed QKV Linear output); lens int64 device [B] with 1 <= lens[b] <= L (key j is visible iff
    j < lens[b]) -> [B, L, heads*64]."""
    qkv = _c(qkv.detach())
    B, T, ld = qkv.shape
    D = heads * 64
    assert ld >= 3 * D and lens.dtype == torch.int64 and lens.is_cuda and lens.numel() == B, (qkv.shape, heads, lens.dtype)
    o = torch.empty((B, T, D), device=qkv.device, dtype=torch.float32)
    base = qkv.data_ptr()
    _call_f("evk_attn_pad_fwd", 4.0 * B * heads * T * T * 64, ctypes.c_void_p(base), ctypes.c_void_p(base + 4 * D),
            ctypes.c_void_p(base + 8 * D), ld, _p(o), D, B, heads, T, _p(lens.contiguous()), ctypes.c_float(scale))
    return o


# ------------------------------------------------------------------------------------------------
# VQ, losses, mel
# ------------------------------------------------------------------------------------------------
def conv_k2s2_fp32(x, weight, bias):
    """Conv1d(kernel 2, stride 2) in exact fp32 FMA arithmetic (no tensor cores): the frozen quantizer's input projection
    (models.py:911-921).  Token indices must not depend on operand rounding -- at the benchmarked shapes the closest
    runner-up codeword is 5e-6 (relative) away, inside TF32 and even 3xTF32 error.  In channels-last memory two
    consecutive frames ARE one row of 2C values, so the conv is a plain [rows, 2C] x [N, 2C]^T product.  No gradient."""
    x = x.detach().contiguous()
    B, T, C = x.shape
    assert T % 2 == 0
    N = weight.shape[0]
    w2 = weight.detach().permute(0, 2, 1).reshape(N, 2 * C).contiguous()             # [n][tap][c]
    y = torch.empty((B, T // 2, N), device=x.device, dtype=torch.float32)
    _call("evk_sgemm_nt_f32", _p(x), 2 * C, _p(w2), 2 * C, _p(y), N, B * (T // 2), N, 2 * C)
    if bias is not None:
        vb = bias.detach().reshape(1, N).expand(B, N).contiguous()
        out = torch.empty_like(y)
        _call("evk_add_bvec", _p(y), N, _p(vb), N, _p(out), N, B, T // 2, N)
        y = out
    return y


def vq_nearest(x, embed):
    """x [B, T, D] channels-last, embed [K, D] -> codes int64 [B, T] (no gradient: frozen quantizer)."""
    x = _cl(x.detach())
    rows, D, ldx = _rows(x)
    embed = embed.detach().contiguous()
    K = embed.shape[0]
    dots = torch.empty((rows, K), device=x.device, dtype=torch.float32)
    _call("evk_sgemm_nt_f32", _p(x), ldx, _p(embed), D, _p(dots), K, rows, K, D)
    codes = torch.empty(x.shape[:-1], device=x.device, dtype=torch.int64)
    scratch = torch.empty(K, device=x.device, dtype=torch.float32)
    _call("evk_vq_argmax", _p(dots), K, _p(x), ldx, _p(embed), D, rows, K, D, _p(codes), _p(scratch))
    return codes


# ---- trainable quantizer (freeze_quantizer: false) ---------------------------------------------
class _SslProjFn(torch.autograd.Function):
    """ssl_proj (Conv1d kernel 2, stride 2) with the exact-fp32 forward of conv_k2s2_fp32 and a TF32 weight gradient:
    dW2 [N, 2C] = dY^T X2 with X2 = the [rows, 2C] view of ssl (two frames per row), on the TMA-fed GEMM."""

    @staticmethod
    def forward(ctx, ssl, weight, bias):
        ctx.save_for_backward(ssl)
        ctx.wshape = weight.shape
        return conv_k2s2_fp32(ssl, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        (ssl,) = ctx.saved_tensors
        N, C, _ = ctx.wshape
        dy = dy.contiguous()
        rows = dy.shape[0] * dy.shape[1]
        x2 = ssl.contiguous().reshape(rows, 2 * C)
        d2 = dy.reshape(rows, N)
        rows4 = (rows + 3) // 4 * 4                                   # the GEMM's K (= rows) pitch must be 16-byte aligned
        if rows4 != rows:
            x2 = torch.nn.functional.pad(x2, (0, 0, 0, rows4 - rows))
            d2 = torch.nn.functional.pad(d2, (0, 0, 0, rows4 - rows))
        dyt = to_channels_first(d2.unsqueeze(0))[0]                  # [N, rows]
        xt = to_channels_first(x2.unsqueeze(0))[0]                   # [2C, rows]
        dw2 = gemm_tf32(dyt, xt)                                     # [N, 2C] = [n][tap][c]
        dw = dw2.reshape(N, 2, C).permute(0, 2, 1).contiguous()      # weight layout [n][c][tap]
        db = torch.empty(N, device=dy.device, dtype=torch.float32)
        _call("evk_col_sum", _p(d2), rows4, N, _p(db))
        return None, dw, db


def ssl_proj_fp32(ssl, weight, bias):
    """conv_k2s2_fp32 with gradients for weight / bias (the unfrozen quantizer's input projection)."""
    return _SslProjFn.apply(ssl, weight, bias)


def vq_kmeans_init_(x, rows_ref, embed, embed_avg, cluster_size, inited, iters=50, idx=None, tag="vq.kmeans"):
    """init_embed_ (core_vq.py:141-149) on the device: k-means over the first min(500, rows) valid rows of x [B, T2, D]
    (rows_ref: device int32 [1] = valid frames per batch row); sets embed = embed_avg = means, cluster_size = bins,
    inited = 1.  idx (int64 [K], optional) replaces the Philox draw of the initial means.  -> the sample indices used."""
    x = _c(x.detach())
    B, T2, D = x.shape
    K = embed.shape[0]
    dev = x.device
    samples = torch.empty((500, D), device=dev, dtype=torch.float32)
    nsamp = torch.empty(1, device=dev, dtype=torch.int32)
    means = torch.empty((K, D), device=dev, dtype=torch.float32)
    idx_out = torch.empty(K, device=dev, dtype=torch.int64)
    if idx is not None:
        idx = idx.to(device=dev, dtype=torch.int64).contiguous()
    _call("evk_vq_kmeans_draw", _p(x), D, B, T2, _p(rows_ref), K, D, _p(idx), _p(rng_state(dev)), ctypes.c_uint64(stream_id(tag)),
          _p(samples), _p(nsamp), _p(means), _p(idx_out))
    buckets = torch.empty(500, device=dev, dtype=torch.int32)
    bins = torch.zeros(K, device=dev, dtype=torch.float32)
    for _ in range(iters):
        _call("evk_vq_kmeans_iter", _p(samples), _p(nsamp), _p(means), K, D, _p(buckets), _p(bins))
    embed.copy_(means)
    embed_avg.copy_(means)
    cluster_size.copy_(bins)
    inited.fill_(1.0)
    return idx_out


def vq_ema_(x, codes, rows_ref, cluster_size, embed_avg, embed, decay=0.99, eps=1e-5):
    """EMA codebook update of EuclideanCodebook.forward in training mode (core_vq.py:218-226), in place."""
    x = _c(x.detach())
    B, T2, D = x.shape
    _call("evk_vq_ema", _p(x), D, _p(codes.contiguous()), B, T2, _p(rows_ref), _p(cluster_size), _p(embed_avg), _p(embed),
          embed.shape[0], D, ctypes.c_float(decay), ctypes.c_float(eps))


class _VqStraightThroughFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, q, rows_ref):
        x = _c(x)
        q = _c(q.detach())
        B, T2, D = x.shape
        y = torch.empty((B, 2 * T2, D), device=x.device, dtype=torch.float32)
        qst = torch.empty((B, T2, D), device=x.device, dtype=torch.float32)
        loss = torch.empty(1, device=x.device, dtype=torch.float32)
        _call("evk_vq_st_fwd", _p(x), D, _p(q), D, B, T2, D, _p(rows_ref), _p(y), _p(qst), _p(loss))
        ctx.save_for_backward(x, qst, rows_ref)
        return y, loss[0]

    @staticmethod
    def backward(ctx, dy, dloss):
        x, qst, rows_ref = ctx.saved_tensors
        B, T2, D = x.shape
        dy = torch.zeros((B, 2 * T2, D), device=x.device, dtype=torch.float32) if dy is None else dy.contiguous()
        g = torch.zeros(1, device=x.device, dtype=torch.float32) if dloss is None else dloss.reshape(1).contiguous()
        dx = torch.empty_like(x)
        _call("evk_vq_st_bwd", _p(dy), _p(x), D, _p(qst), B, T2, D, _p(rows_ref), _p(g), _p(dx))
        return dx, None, None


def vq_straight_through(x, q, rows_ref):
    """VectorQuantization.forward in training mode (core_vq.py:308-316) + the nearest x2 upsample (models.py:924-927):
    x [B, T2, D] (differentiable), q = its codewords -> (x + (q - x) upsampled to [B, 2*T2, D],
    commit loss = mean((x + (q - x) - x)^2) over the rows t < rows_ref)."""
    return _VqStraightThroughFn.apply(x, q, rows_ref)


class _ReduceLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, kind, scale_):
        a = a.contiguous()
        b = b.contiguous() if b is not None else None
        out = torch.zeros(1, device=a.device, dtype=torch.float32)
        _call("evk_reduce_loss", kind, _p(a), _p(b), a.numel(), ctypes.c_float(scale_), _p(out))
        ctx.save_for_backward(a, b)
        ctx.k = (kind, scale_)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        kind, scale_ = ctx.k
        g = g.reshape(1).contiguous()
        da = torch.empty_like(a)
        _call("evk_reduce_loss_bwd", kind, _p(a), _p(b), a.numel(), ctypes.c_float(scale_), _p(g), _p(da))
        return da, None, None, None


def mean_sq_one_minus(a):
    """mean((1 - a)^2)"""
    return _ReduceLossFn.apply(a, None, 0, 1.0 / a.numel())


def mean_sq(a):
    return _ReduceLossFn.apply(a, None, 1, 1.0 / a.numel())


def mean_abs_diff(a, b):
    """mean(|a - b|), gradient wrt a only (b is the detached target)."""
    return _ReduceLossFn.apply(a, b.detach(), 2, 1.0 / a.numel())


class _KlFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z_p, logs_q, m_p, logs_p, length, inv_norm):
        ts = [_cl(t) for t in (z_p, logs_q, m_p, logs_p)]
        B, T, C = ts[0].shape
        out = torch.zeros(1, device=ts[0].device, dtype=torch.float32)
        _call("evk_kl_loss", _p(ts[0]), _rows(ts[0])[2], _p(ts[1]), _rows(ts[1])[2], _p(ts[2]), _rows(ts[2])[2], _p(ts[3]),
              _rows(ts[3])[2], B, T, C, _p(length), _p(out))
        ctx.save_for_backward(*ts, inv_norm)
        ctx.length = length
        return out[0] * inv_norm

    @staticmethod
    def backward(ctx, g):
        z_p, logs_q, m_p, logs_p, inv_norm = ctx.saved_tensors
        B, T, C = z_p.shape
        gg = (g * inv_norm).reshape(1).contiguous()
        outs = [torch.empty((B, T, C), device=z_p.device, dtype=torch.float32) for _ in range(4)]
        _call("evk_kl_loss_bwd", _p(z_p), _rows(z_p)[2], _p(logs_q), _rows(logs_q)[2], _p(m_p), _rows(m_p)[2], _p(logs_p),
              _rows(logs_p)[2], B, T, C, _p(ctx.length), _p(gg), ctypes.c_float(1.0), _p(outs[0]), _p(outs[1]), _p(outs[2]),
              _p(outs[3]), C)
        return outs[0], outs[1], outs[2], outs[3], None, None


def kl_loss(z_p, logs_q, m_p, logs_p, length):
    """losses.py:46-61 on channels-last tensors; length int32 [B] (mask = t < length)."""
    C = z_p.shape[-1]
    inv_norm = 1.0 / (length.sum().to(torch.float32))        # sum(z_mask) over [B,1,T]
    return _KlFn.apply(z_p, logs_q, m_p, logs_p, length, inv_norm)


# ---- mel ---------------------------------------------------------------------------------------
class MelBank:
    """Slaney filterbank (librosa.filters.mel restated; see mel_processing.slaney_filterbank) in CSR-by-mel form."""
    _cache = {}

    def __init__(self, fb, device):
        import numpy as np
        n_mels, n_bins = fb.shape
        ptr, idx, val = [0], [], []
        for m in range(n_mels):
            nz = np.nonzero(fb[m])[0]
            idx.extend(nz.tolist())
            val.extend(fb[m, nz].tolist())
            ptr.append(len(idx))
        self.n_mels, self.n_bins = n_mels, n_bins
        self.ptr = torch.tensor(ptr, dtype=torch.int32, device=device)
        self.idx = torch.tensor(idx, dtype=torch.int32, device=device)
        self.val = torch.tensor(val, dtype=torch.float32, device=device)


def stft_frames(L, n_fft, hop, pad):
    return (L + 2 * pad - n_fft) // hop + 1


class _MelFn(torch.autograd.Function):
    """|X| / log-mel of reflect-padded frames.  geo = (n_fft, hop, win, pad): the training configuration (2048, hop, 2048,
    (2048 - hop) / 2) runs on the warp-per-frame register-FFT kernel, everything else on the general kernel of stft.cu."""

    @staticmethod
    def forward(ctx, wav, bank, geo, want_spec, want_mel, lens):
        n_fft, hop, win, pad = geo
        wav = wav.contiguous()
        B, Lw = wav.shape
        assert bank.n_bins == n_fft // 2 + 1
        T = stft_frames(Lw, n_fft, hop, pad)
        need_grad = ctx.needs_input_grad[0]
        ld_spec = (bank.n_bins + 3) // 4 * 4          # 16-byte row pitch so |X| can feed the tensor-core GEMMs directly
        spec = (torch.zeros if ld_spec != bank.n_bins else torch.empty)((B, T, ld_spec), device=wav.device, dtype=torch.float32) if want_spec else None
        mel = torch.empty((B, T, bank.n_mels), device=wav.device, dtype=torch.float32) if want_mel else None
        cplx = torch.empty((B, T, bank.n_bins, 2), device=wav.device, dtype=torch.float32) if need_grad else None
        if n_fft == 2048 and win == 2048 and pad == (2048 - hop) // 2:
            _call("evk_mel_fwd", _p(wav), _p(lens), B, Lw, Lw, hop, bank.n_mels, _p(bank.ptr), _p(bank.idx), _p(bank.val), _p(spec),
                  ld_spec, _p(mel), bank.n_mels, _p(cplx))
        else:
            _call("evk_stft_fwd", _p(wav), _p(lens), B, Lw, Lw, n_fft, hop, win, pad, T, ctypes.c_float(1e-6), _p(cplx), _p(spec), ld_spec,
                  bank.n_mels, _p(bank.ptr), _p(bank.idx), _p(bank.val), ctypes.c_float(1e-5), _p(mel), bank.n_mels)
        ctx.k = (bank, geo, B, Lw, T, lens)
        ctx.save_for_backward(cplx, mel)
        if spec is None:
            spec = torch.empty(0, device=wav.device)
        else:
            spec = spec[:, :, :bank.n_bins]
        if mel is None:
            mel = torch.empty(0, device=wav.device)
        ctx.mark_non_differentiable(spec)
        return spec, mel

    @staticmethod
    def backward(ctx, _dspec, dmel):
        bank, (n_fft, hop, win, pad), B, Lw, T, lens = ctx.k
        cplx, mel = ctx.saved_tensors
        dmel = dmel.contiguous()
        dwav = torch.zeros((B, Lw), device=dmel.device, dtype=torch.float32)
        _call("evk_stft_bwd", None, _p(dmel), bank.n_mels, _p(cplx), _p(mel), bank.n_mels, ctypes.c_float(1e-6), ctypes.c_float(1e-5),
              bank.n_mels, _p(bank.ptr), _p(bank.idx), _p(bank.val), _p(lens), B, Lw, Lw, n_fft, hop, win, pad, T, _p(dwav))
        return dwav, None, None, None, None, None


def mel_frontend(wav, bank, hop, want_spec=False, want_mel=True, lens=None, n_fft=2048, win=None, pad=None):
    """wav [B, L] -> (spec [B,T,n_fft/2+1] or None, log-mel [B,T,n_mels] or None), channels-last; differentiable wrt wav via mel.
    lens (int32 [B], optional): per-row valid length (reflection at each row's own end, zero frames past it)."""
    win = n_fft if win is None else win
    pad = (n_fft - hop) // 2 if pad is None else pad
    spec, mel = _MelFn.apply(wav, bank, (n_fft, hop, win, pad), want_spec, want_mel, lens)
    return (spec if want_spec else None), (mel if want_mel else None)


class _StftFn(torch.autograd.Function):
    """complex STFT [B, T, n_fft/2+1, 2] of reflect-padded frames (torch.stft(return_complex=True) semantics when
    pad = n_fft / 2), differentiable wrt wav."""

    @staticmethod
    def forward(ctx, wav, n_fft, hop, win, pad):
        wav = wav.contiguous()
        B, Lw = wav.shape
        T = stft_frames(Lw, n_fft, hop, pad)
        out = torch.empty((B, T, n_fft // 2 + 1, 2), device=wav.device, dtype=torch.float32)
        _call("evk_stft_fwd", _p(wav), None, B, Lw, Lw, n_fft, hop, win, pad, T, ctypes.c_float(0.0), _p(out), None, 0, 0, None, None, None,
              ctypes.c_float(0.0), None, 0)
        ctx.k = (n_fft, hop, win, pad, B, Lw, T)
        return out

    @staticmethod
    def backward(ctx, g):
        n_fft, hop, win, pad, B, Lw, T = ctx.k
        g = g.contiguous()
        dwav = torch.zeros((B, Lw), device=g.device, dtype=torch.float32)
        _call("evk_stft_bwd", _p(g), None, 0, None, None, 0, ctypes.c_float(0.0), ctypes.c_float(0.0), 0, None, None, None, None, B, Lw, Lw,
              n_fft, hop, win, pad, T, _p(dwav))
        return dwav, None, None, None, None


def stft(wav, n_fft, hop, win=None, center=True):
    """wav [B, L] -> [B, T, n_fft/2+1, 2] (re, im).  center=True: torch.stft defaults (reflect pad n_fft/2, T = 1 + L // hop);
    center=False: no padding.  Window: periodic Hann(win) centred in the n_fft frame."""
    win = n_fft if win is None else win
    return _StftFn.apply(wav, n_fft, hop, win, n_fft // 2 if center else 0)


class _CplxL1Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        n = a.numel() // 2
        loss = torch.zeros(1, device=a.device, dtype=torch.float32)
        grad = torch.empty_like(a) if ctx.needs_input_grad[0] else None
        _call("evk_cplx_l1", _p(a), _p(b), n, ctypes.c_float(1.0 / n), _p(loss), _p(grad))
        ctx.save_for_backward(grad)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None


def complex_l1(a, b):
    """F.l1_loss(a, b) for complex tensors stored as [..., 2]: mean modulus of the difference; gradient wrt a only."""
    return _CplxL1Fn.apply(a, b.detach())


def mrstft_loss(y_hat, y, windows=(4096, 2048, 1024, 512, 256), hop=147, n_fft_min=2048):
    """Multi-resolution STFT loss exactly as the reference defines it (bs_roformer.py:565-581): sum over window sizes of the
    complex L1 between torch.stft(n_fft=max(win, 2048), hop=147, win_length=win, hann, center=True) of both signals.
    y_hat, y: [B, L].  An opt-in extension of the stage-2 generator loss (BASELINE config 5); not part of SovitsTrain parity."""
    total = 0
    for w in windows:
        n_fft = max(w, n_fft_min)
        total = total + complex_l1(stft(y_hat, n_fft, hop, w), stft(y.detach(), n_fft, hop, w))
    return total


def spec_to_mel(spec, bank):
    """|X| [B, T, 1025] channels-last -> log-mel [B, T, 128] (no gradient: applied to ground-truth features)."""
    spec = _cl(spec.detach())
    rows, F, ld = _rows(spec)
    mel = torch.empty((*spec.shape[:-1], bank.n_mels), device=spec.device, dtype=torch.float32)
    _call("evk_spec_to_mel", _p(spec), rows, ld, bank.n_mels, _p(bank.ptr), _p(bank.idx), _p(bank.val), _p(mel), bank.n_mels)
    return mel


# ---- optimiser -----------------------------------------------------------------------------------
def adamw_flat(p, g, m, v, hyper, lr_scale, betas, eps, wd, grad_scale=1.0, gnorm_sq=None):
    """hyper: device float32 [lr, step] (step already incremented for this update)."""
    _call("evk_adamw_flat", _p(p), _p(g), _p(m), _p(v), p.numel(), _p(hyper), ctypes.c_float(lr_scale),
          ctypes.c_float(betas[0]), ctypes.c_float(betas[1]), ctypes.c_float(eps), ctypes.c_float(wd),
          ctypes.c_float(grad_scale), _p(gnorm_sq))


def scalar_add(x, v):
    _call("evk_scalar_add", _p(x), ctypes.c_float(v))


# ------------------------------------------------------------------------------------------------
# stage-1 AR GPT (t2s_model.py:431-490)
# ------------------------------------------------------------------------------------------------
class _FlashAttnFn(torch.autograd.Function):
    """fused prefix-LM self-attention on the packed in_proj output qkv [B, L, 3D]."""

    @staticmethod
    def forward(ctx, qkv, cfg):
        H, X, xlen, ylen, scale_, p_drop, sid = cfg
        qkv = qkv.contiguous()
        B, Lq, D3 = qkv.shape
        D = D3 // 3
        dk = D // H
        out = torch.empty((B, Lq, D), device=qkv.device, dtype=torch.float32)
        lse = torch.empty((B * H, Lq), device=qkv.device, dtype=torch.float32)
        base = qkv.data_ptr()
        _call("evk_flash_attn_fwd", base, base + 4 * D, base + 8 * D, D3, _p(out), D, _p(lse), B, H, Lq, X, dk, _p(xlen), _p(ylen),
              ctypes.c_float(scale_), ctypes.c_float(p_drop), _p(rng_state(qkv.device)), ctypes.c_uint64(sid))
        ctx.cfg = cfg
        ctx.save_for_backward(qkv, out, lse)
        return out

    @staticmethod
    def backward(ctx, dout):
        H, X, xlen, ylen, scale_, p_drop, sid = ctx.cfg
        qkv, out, lse = ctx.saved_tensors
        B, Lq, D3 = qkv.shape
        D = D3 // 3
        dk = D // H
        dout = dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse)
        base, dbase = qkv.data_ptr(), dqkv.data_ptr()
        _call("evk_flash_attn_bwd", base, base + 4 * D, base + 8 * D, D3, _p(out), D, _p(lse), _p(dout), D, _p(delta),
              dbase, dbase + 4 * D, dbase + 8 * D, D3, B, H, Lq, X, dk, _p(xlen), _p(ylen), ctypes.c_float(scale_),
              ctypes.c_float(p_drop), _p(rng_state(qkv.device)), ctypes.c_uint64(sid))
        return dqkv, None


def flash_attention(qkv, *, heads, prefix, xlen, ylen, p_drop=0.0, tag="gpt.attn"):
    """softmax(q k^T / sqrt(dk) + prefix-LM mask) v with optional probability dropout; qkv = in_proj(x) [B, L, 3D]."""
    dk = qkv.shape[-1] // 3 // heads
    cfg = (heads, int(prefix), xlen, ylen, 1.0 / math.sqrt(dk), float(p_drop), stream_id(tag))
    return _FlashAttnFn.apply(qkv, cfg)


class _GptEmbedFn(torch.autograd.Function):
    """h = cat([xe + ax * pe[:X], ye + ay * pe[:Y]], dim=1)  (embedding.py:71-81 twice + t2s_model.py:462)."""

    @staticmethod
    def forward(ctx, xe, ye, ax, ay, pe):
        xe, ye = xe.contiguous(), ye.contiguous()
        B, X, D = xe.shape
        Y = ye.shape[1]
        Lq = X + Y
        h = torch.empty((B, Lq, D), device=xe.device, dtype=torch.float32)
        _call("evk_sinepos_add", _p(xe), D, X * D, _p(pe), D, _p(ax), h.data_ptr(), D, Lq * D, B, X, D)
        _call("evk_sinepos_add", _p(ye), D, Y * D, _p(pe), D, _p(ay), h.data_ptr() + 4 * X * D, D, Lq * D, B, Y, D)
        ctx.save_for_backward(pe)
        ctx.k = (B, X, Y, D)
        return h

    @staticmethod
    def backward(ctx, dh):
        (pe,) = ctx.saved_tensors
        B, X, Y, D = ctx.k
        dh = dh.contiguous()
        Lq = X + Y
        da = torch.zeros(2, device=dh.device, dtype=torch.float32)
        _call("evk_sinepos_bwd", dh.data_ptr(), D, Lq * D, _p(pe), D, da.data_ptr(), B, X, D)
        _call("evk_sinepos_bwd", dh.data_ptr() + 4 * X * D, D, Lq * D, _p(pe), D, da.data_ptr() + 4, B, Y, D)
        return dh[:, :X], dh[:, X:], da[0:1], da[1:2], None


def gpt_embed(xe, ye, alpha_x, alpha_y, pe):
    return _GptEmbedFn.apply(xe, ye, alpha_x, alpha_y, pe)


class _CeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, targets, topk, ignore, V, count):
        logits = _cl(logits)
        rows, Vp, ld = _rows(logits)
        targets = targets.contiguous()
        dev = logits.device
        T = _count_period(logits, count)
        lse = torch.empty(rows, device=dev, dtype=torch.float32)
        nll = torch.empty(rows, device=dev, dtype=torch.float32)
        flags = torch.empty(rows, device=dev, dtype=torch.uint8)
        out2 = torch.empty(2, device=dev, dtype=torch.float32)
        _call("evk_ce_fwd", _p(logits), ld, _p(targets), rows, V, topk, ignore, _p(count), T, _p(lse), _p(nll), _p(flags), _p(out2))
        ctx.save_for_backward(logits, targets, lse, count)
        ctx.V, ctx.T = V, T
        ctx.mark_non_differentiable(out2)
        return out2[0].clone(), out2

    @staticmethod
    def backward(ctx, gloss, _g2):
        logits, targets, lse, count = ctx.saved_tensors
        rows, Vp, ld = _rows(logits)
        V = ctx.V
        gl = gloss.reshape(1).contiguous().float()
        dl = (torch.empty if Vp == V else torch.zeros)(logits.shape, device=logits.device, dtype=torch.float32)
        _call("evk_ce_bwd", _p(logits), ld, _p(targets), _p(lse), _p(gl), rows, _p(count), ctx.T, _p(dl), Vp, rows, V)
        return dl, None, None, None, None, None


def _count_period(logits, count):
    """-> T, the positions per batch row of [B, T, Vp] logits that a counted-length bound `count` refers to (1 without one)."""
    if count is None:
        return 1
    assert logits.dim() == 3, "a counted length needs [B, T, V] logits"
    assert count.dtype == torch.int32 and count.is_cuda and count.numel() == 1, "count: one int32 device value"
    return logits.shape[1]


def attn_decode_dev(cache, n_prev_dev, heads, row, skip=None):
    """Graph-replayable token step: append `row` [B, 1, 3 * heads * 32] at index *n_prev_dev (int32 device scalar) of the cache
    and attend rows 0 .. *n_prev_dev.  -> [B, 1, heads * 32].  skip: optional int32 device [B, 2]; item b then leaves out the
    keys skip[b, 0] .. skip[b, 1] - 1 (its text padding in a batch padded to a common text length)."""
    assert cache.dim() == 3 and cache.stride(2) == 1 and cache.shape[2] == 3 * heads * 32 and n_prev_dev.dtype == torch.int32
    assert skip is None or (skip.dtype == torch.int32 and skip.is_contiguous() and tuple(skip.shape) == (cache.shape[0], 2))
    B, W = cache.shape[0], cache.shape[2]
    row = row.contiguous()
    _call("evk_cache_append", _p(row), W, _p(cache), cache.stride(0), cache.stride(1), _p(n_prev_dev), B, W)
    out = torch.empty((B, 1, heads * 32), device=cache.device, dtype=torch.float32)
    _call("evk_attn_decode_dev", _p(cache), cache.stride(0), cache.stride(1), _p(n_prev_dev), _p(skip), B, heads,
          ctypes.c_float(1.0 / math.sqrt(32.0)), _p(out), heads * 32)
    return out


def attn_decode_h16(cache, n_prev_dev, heads, row, skip=None):
    """attn_decode_dev on a 16-bit K/V cache [B, rows, 2 * heads * 32] (fp16 or bf16, k then v; evk_attn_decode_h16): the k and v
    of `row` [B, 1, 3 * heads * 32] fp32 (the step's in_proj output) are rounded to nearest even into cache row *n_prev_dev, and
    rows 0 .. *n_prev_dev are attended with row's fp32 q.  -> [B, 1, heads * 32] fp32.  One launch, graph-replayable."""
    assert cache.dim() == 3 and cache.stride(2) == 1 and cache.shape[2] == 2 * heads * 32 and cache.dtype in H16_TYPES
    assert n_prev_dev.dtype == torch.int32 and row.dtype == torch.float32 and row.shape[-1] == 3 * heads * 32
    assert skip is None or (skip.dtype == torch.int32 and skip.is_contiguous() and tuple(skip.shape) == (cache.shape[0], 2))
    B = cache.shape[0]
    row = row.reshape(B, -1).contiguous()
    out = torch.empty((B, 1, heads * 32), device=cache.device, dtype=torch.float32)
    _call("evk_attn_decode_h16", _p(row), row.stride(0), _p(cache), cache.stride(0), cache.stride(1),
          int(cache.dtype == torch.bfloat16), _p(n_prev_dev), _p(skip), B, heads, ctypes.c_float(1.0 / math.sqrt(32.0)), _p(out),
          heads * 32)
    return out


def sample_tokens(logits, V, eos, icfg, fcfg, n_dev, hist, seen, fin, emb, pe, alpha, x_next, q=None, eos_steps=1):
    """One fused sampling step over the rows of `logits` [B, >= V] (evk_sample_tokens; see include/evk.h for the buffers).
    EOS is excluded at the steps idx < eos_steps (1: infer_panel_batch_infer; 11: infer_panel_naive and prompt-free decoding).
    Everything it reads or writes stays in device memory, so it can be part of a captured CUDA graph."""
    B, D = logits.shape[0], x_next.shape[-1]
    if int(eos_steps) != eos_steps or eos_steps < 0:
        raise ValueError(f"sample_tokens: eos_steps must be an integer >= 0, got {eos_steps!r}")
    assert logits.stride(-1) == 1 and hist.dtype == torch.int64 and seen.dtype == torch.int32 and fin.dtype == torch.int32
    assert icfg.dtype == torch.int64 and fcfg.dtype == torch.float32 and x_next.is_contiguous() and pe.is_contiguous()
    assert q is None or (q.shape[0] == B and q.stride(-1) == 1)
    _call("evk_sample_tokens", _p(logits), logits.stride(0), B, V, eos, int(eos_steps), _p(icfg), _p(fcfg), _p(n_dev), _p(q),
          q.stride(0) if q is not None else 0, _p(hist), hist.stride(0), _p(seen), _p(fin), _p(emb), _p(pe), _p(alpha),
          _p(x_next), D)


def sample_tokens_rows(logits, V, eos, icfg, fcfg, n_dev, hist, seen, fin, emb, pe, alpha, x_next):
    """sample_tokens with one configuration per row (evk_sample_tokens_rows): icfg int64 [B, 8] = (seed, prefix, n0, top_k,
    early_stop, max_steps, eos_steps, key row), fcfg float32 [B, 4] = (top_p, temperature, penalty, unused)."""
    B, D = logits.shape[0], x_next.shape[-1]
    assert logits.stride(-1) == 1 and hist.dtype == torch.int64 and seen.dtype == torch.int32 and fin.dtype == torch.int32
    assert icfg.dtype == torch.int64 and icfg.is_contiguous() and tuple(icfg.shape) == (B, 8)
    assert fcfg.dtype == torch.float32 and fcfg.is_contiguous() and tuple(fcfg.shape) == (B, 4)
    assert x_next.is_contiguous() and pe.is_contiguous()
    _call("evk_sample_tokens_rows", _p(logits), logits.stride(0), B, V, eos, _p(icfg), _p(fcfg), _p(n_dev), _p(hist),
          hist.stride(0), _p(seen), _p(fin), _p(emb), _p(pe), _p(alpha), _p(x_next), D)


def ce_sum_topk(logits, targets, topk=3, ignore_index=1024, V=None, count=None):
    """-> (sum cross-entropy (differentiable), device float32 [2] = (loss, top-k accuracy ignoring ignore_index)).
    V: number of real classes when the last dim of `logits` is zero-padded.  count: None, or an int32 device scalar n for
    [B, T, Vp] logits: positions t >= n of every row add no loss, no accuracy count and no gradient (evk_ce_fwd)."""
    loss, out2 = _CeFn.apply(logits, targets, int(topk), int(ignore_index), int(V or logits.shape[-1]), count)
    return loss, out2


class _DpoCeFn(torch.autograd.Function):
    """loss_1 + loss_2 of Text2SemanticDecoder.forward (t2s_model.py:417-427) from chosen / rejected logits."""

    @staticmethod
    def forward(ctx, lc, tc, lr_, tr, topk, ignore, V, beta, count):
        lc, lr_ = _cl(lc), _cl(lr_)
        B, Yc = tc.shape
        Yr = tr.shape[1]
        dev = lc.device
        tc, tr = tc.reshape(-1).contiguous(), tr.reshape(-1).contiguous()
        if count is not None:
            assert count.dtype == torch.int32 and count.is_cuda and count.numel() == 2, "count: int32 device (chosen, rejected)"
        cnt = (None, None) if count is None else (count[0:1], count[1:2])
        bufs = []
        for lg, tg, rows, T, cn in ((lc, tc, B * Yc, Yc, cnt[0]), (lr_, tr, B * Yr, Yr, cnt[1])):
            lse = torch.empty(rows, device=dev, dtype=torch.float32)
            nll = torch.empty(rows, device=dev, dtype=torch.float32)
            flags = torch.empty(rows, device=dev, dtype=torch.uint8)
            o2 = torch.empty(2, device=dev, dtype=torch.float32)
            _call("evk_ce_fwd", _p(lg), _rows(lg)[2], _p(tg), rows, V, topk, ignore, _p(cn), T, _p(lse), _p(nll), _p(flags), _p(o2))
            bufs.append((lse, nll, o2))
        out3 = torch.empty(3, device=dev, dtype=torch.float32)
        coef = torch.empty((2, B), device=dev, dtype=torch.float32)
        _call("evk_dpo_head", _p(bufs[0][1]), Yc, _p(cnt[0]), _p(bufs[1][1]), Yr, _p(cnt[1]), B, ctypes.c_float(beta), _p(out3),
              _p(coef[0]), _p(coef[1]))
        ctx.save_for_backward(lc, tc, bufs[0][0], lr_, tr, bufs[1][0], coef, count)
        ctx.k = (B, Yc, Yr, V)
        metrics = torch.stack([out3[0], out3[1], bufs[0][2][1]])        # (loss_1, loss_2, top-k acc of the chosen branch)
        ctx.mark_non_differentiable(metrics)
        return out3[2].clone(), metrics

    @staticmethod
    def backward(ctx, g, _gm):
        lc, tc, lsec, lr_, tr, lser, coef, count = ctx.saved_tensors
        B, Yc, Yr, V = ctx.k
        gc = _AxpbyFn_scale(coef, g)
        cnt = (None, None) if count is None else (count[0:1], count[1:2])
        outs = []
        for lg, tg, lse, Yn, cf, cn in ((lc, tc, lsec, Yc, gc[0], cnt[0]), (lr_, tr, lser, Yr, gc[1], cnt[1])):
            rows, Vp, ld = _rows(lg)
            dl = (torch.empty if Vp == V else torch.zeros)(lg.shape, device=lg.device, dtype=torch.float32)
            _call("evk_ce_bwd", _p(lg), ld, _p(tg), _p(lse), _p(cf), Yn, _p(cn), Yn, _p(dl), Vp, rows, V)
            outs.append(dl)
        return outs[0], None, outs[1], None, None, None, None, None, None


def _AxpbyFn_scale(coef, g):
    """coef * g for a device scalar g (tiny [2, B] tensor)."""
    return (coef * g.reshape(1, 1)).contiguous()


def dpo_ce(logits_c, targets_c, logits_r, targets_r, topk=3, ignore_index=1024, V=None, beta=0.2, count=None):
    """-> (loss_1 + loss_2 (differentiable), device [3] = (loss_1, loss_2, top-k acc)).  count: None, or int32 device [2] =
    (chosen, rejected) counted lengths: positions at or past a branch's count add no loss, accuracy or gradient, and do not
    enter that branch's log-prob sums (evk_ce_fwd / evk_dpo_head)."""
    return _DpoCeFn.apply(logits_c, targets_c, logits_r, targets_r, int(topk), int(ignore_index),
                          int(V or logits_c.shape[-1]), float(beta), count)


def dpo_reject_rows(y, spans, yc, width):
    """Rejected rows of the DPO variant on the device (evk_dpo_reject_rows) -> (rows int64 [B, width], lens int64 [B]):
    row b = y[b, :i0] ++ y[b, i0:i1] ++ y[b, i0:i1] ++ y[b, i1:Yc], zero after, with (i0, i1) = spans[b] (int32 device
    [B, 2]) and Yc = yc (int32 device scalar).  width must hold the longest row (Yc + max(i1 - i0)).  No host sync."""
    assert y.dtype == torch.int64 and y.dim() == 2 and y.stride(1) == 1 and y.is_cuda
    assert spans.dtype == torch.int32 and spans.is_contiguous() and tuple(spans.shape) == (y.shape[0], 2)
    assert yc.dtype == torch.int32 and yc.numel() == 1
    B = y.shape[0]
    out = torch.empty((B, int(width)), device=y.device, dtype=torch.int64)
    lens = torch.empty(B, device=y.device, dtype=torch.int64)
    _call("evk_dpo_reject_rows", _p(y), y.stride(0), B, _p(spans), _p(yc), _p(out), int(width), _p(lens))
    return out, lens


def scaled_adam(st, gscale=1.0, zero_grad=True):
    """one ScaledAdam update over the arenas held by `st` (train/gpt_step.FlatScaledAdam)."""
    c = st.cfg
    _call("evk_scaled_adam", _p(st.flat_p), _p(st.flat_g), _p(st.flat_delta), _p(st.flat_v), _p(st.chunks), st.chunks.shape[0],
          _p(st.numel), st.numel.shape[0], _p(st.stats), _p(st.rms), _p(st.sv), _p(st.sg), _p(st.coef), _p(st.hyper),
          _p(st.stepbuf), _p(st.norms), _p(st.thr), _p(st.glob), ctypes.c_float(gscale), ctypes.c_float(c["betas"][0]),
          ctypes.c_float(c["betas"][1]), ctypes.c_float(c["clipping_scale"]), int(c["clipping_update_period"]),
          ctypes.c_float(c["scalar_lr_scale"]), ctypes.c_float(c["eps"]), ctypes.c_float(c["param_min_rms"]),
          ctypes.c_float(c["param_max_rms"]), ctypes.c_float(c["scalar_max"]), int(c["size_update_period"]),
          1 if zero_grad else 0)


def gemm_tf32(a, b, out=None, bias=None, res=None, act=ACT_NONE, slope=0.0, splits=1):
    """out[M, N] (+)= a[M, K] @ b[N, K]^T on the TMA-fed wgmma GEMM (no autograd).  splits > 1 accumulates into `out`."""
    M, K = a.shape
    N = b.shape[0]
    assert b.shape[1] == K and a.stride(1) == 1 and b.stride(1) == 1
    if out is None:
        out = (torch.zeros if splits > 1 else torch.empty)((M, N), device=a.device, dtype=torch.float32)
    _call_f("evk_gemm_tf32", 2.0 * M * N * K, _p(a), a.stride(0), _p(b), b.stride(0), _p(out), out.stride(0), M, N, K, _p(bias),
            _p(res), res.stride(0) if res is not None else 0, act, ctypes.c_float(slope), splits)
    return out


# ------------------------------------------------------------------------------------------------
# 2-D convolution family (UVR5 VR separator, uvr5.py): channels-last [B, H, W, pitch] operands
# ------------------------------------------------------------------------------------------------
C2_NONE, C2_RELU, C2_LRELU, C2_SIGMOID = 0, 1, 2, 3


class CLView:
    """Rows r0 .. r0+H and channels c0 .. c0+C of a contiguous channels-last fp32 CUDA buffer [B, Hs, W, pitch]: a layer
    reads or writes a slice of a concat buffer in place."""
    __slots__ = ("buf", "c0", "C", "r0", "H")

    def __init__(self, buf, c0=0, C=None, r0=0, H=None):
        assert buf.dim() == 4 and buf.is_contiguous() and buf.dtype == torch.float32 and buf.is_cuda, (buf.shape, buf.dtype)
        self.buf, self.c0, self.r0 = buf, c0, r0
        self.C = buf.shape[3] - c0 if C is None else C
        self.H = buf.shape[1] - r0 if H is None else H
        assert 0 <= c0 and c0 + self.C <= buf.shape[3] and 0 <= r0 and r0 + self.H <= buf.shape[1], (buf.shape, c0, C, r0, H)

    @property
    def B(self):
        return self.buf.shape[0]

    @property
    def W(self):
        return self.buf.shape[2]

    def args(self):
        """-> (pointer to channel c0 of pixel (0, r0, 0), pixel pitch, batch stride) in the library's argument order"""
        pitch = self.buf.shape[3]
        return (ctypes.c_void_p(self.buf.data_ptr() + 4 * (self.r0 * self.W * pitch + self.c0)), pitch,
                self.buf.stride(0))


def conv2d_out(n, k, stride, pad, dil):
    return (n + 2 * pad - dil * (k - 1) - 1) // stride + 1


def conv2d(x: CLView, w, y: CLView, *, k, stride=1, pad=0, dil=1, scale=None, bias=None, act=C2_NONE):
    """y = act(conv2d(x) * scale + bias) (evk_conv2d_fwd): w [N, k, k, C] fp32 contiguous; y must be [B, Ho, Wo, N].
    pad and dil are ints, or (rows, columns) pairs."""
    N = w.shape[0]
    assert w.is_contiguous() and tuple(w.shape) == (N, k, k, x.C) and y.C == N and y.B == x.B, (w.shape, x.C, y.C)
    (ph, pw), (dh, dw) = [v if isinstance(v, (tuple, list)) else (v, v) for v in (pad, dil)]
    Ho, Wo = conv2d_out(x.H, k, stride, ph, dh), conv2d_out(x.W, k, stride, pw, dw)
    assert (y.H, y.W) == (Ho, Wo), ((y.H, y.W), (Ho, Wo))
    _call_f("evk_conv2d_fwd", 2.0 * x.B * Ho * Wo * N * k * k * x.C, *x.args(), _p(w), _p(scale), _p(bias), *y.args(),
            x.B, x.H, x.W, x.C, N, k, stride, ph, pw, dh, dw, act, tag=f"k{k}")


def pack_conv_h16(w, dtype):
    """Conv weight [N, k, k, C] (the layout conv2d takes) -> PackedH16 [N, k*k*C rounded up to 64] rounded to `dtype`
    (torch.float16 or torch.bfloat16) to nearest even, K = k*k*C, the layout evk_conv2d_fwd_h16 reads.  A weight that is
    already exactly 16-bit keeps its bits."""
    assert w.dim() == 4 and w.shape[1] == w.shape[2], w.shape
    return pack_weight_h16(w.reshape(w.shape[0], -1), dtype)


def conv2d_h16(x: CLView, w, y: CLView, *, k, stride=1, pad=0, dil=1, scale=None, bias=None, act=C2_NONE):
    """conv2d with 16-bit products (evk_conv2d_fwd_h16): h(x) . h(w) accumulated in fp32, then act(acc * scale + bias) in
    fp32.  w: pack_conv_h16 of the [N, k, k, C] weight; the other arguments as for conv2d."""
    N = w.w.shape[0]
    assert w.K == k * k * x.C and y.C == N and y.B == x.B, (w.K, k, x.C, y.C)
    (ph, pw), (dh, dw) = [v if isinstance(v, (tuple, list)) else (v, v) for v in (pad, dil)]
    Ho, Wo = conv2d_out(x.H, k, stride, ph, dh), conv2d_out(x.W, k, stride, pw, dw)
    assert (y.H, y.W) == (Ho, Wo), ((y.H, y.W), (Ho, Wo))
    _call_f("evk_conv2d_fwd_h16", 2.0 * x.B * Ho * Wo * N * k * k * x.C, *x.args(), _p(w.w), w.w.shape[1],
            int(w.w.dtype == torch.bfloat16), _p(scale), _p(bias), *y.args(), x.B, x.H, x.W, x.C, N, k, stride, ph, pw, dh, dw,
            act, tag=f"k{k}")


def dwconv3x3(x: CLView, w, y: CLView, dil):
    """depthwise 3x3, stride 1, padding = dil (evk_dwconv3x3_fwd): w [C, 9]"""
    assert w.is_contiguous() and tuple(w.shape) == (x.C, 9) and (y.B, y.H, y.W, y.C) == (x.B, x.H, x.W, x.C)
    _call("evk_dwconv3x3_fwd", *x.args(), _p(w), *y.args(), x.B, x.H, x.W, x.C, dil)


def resize_bilinear_ac(x: CLView, y: CLView):
    """F.interpolate(mode="bilinear", align_corners=True) from x's extent to y's (evk_resize_bilinear_ac)"""
    assert y.B == x.B and y.C == x.C
    _call("evk_resize_bilinear_ac", *x.args(), x.H, x.W, *y.args(), y.H, y.W, x.B, x.C)


def mean_h(x: CLView):
    """-> [B, 1, W, C] mean over rows (evk_mean_h)"""
    y = torch.empty((x.B, 1, x.W, x.C), device=x.buf.device, dtype=torch.float32)
    _call("evk_mean_h", *x.args(), _p(y), x.B, x.H, x.W, x.C)
    return y


def vr_mask_head(h: CLView, w, mix, offset, split_bin=0, e_lo=1.0, e_hi=1.0, use_agg=False):
    """CascadedASPPNet's mask head (evk_vr_mask_head): h [B, max_bin, W, Ch], w [2, Ch], mix NCHW [B, 2, out_bin, W]
    -> [B, 2, out_bin, W - 2 offset]"""
    B, two, out_bin, W = mix.shape
    assert two == 2 and mix.is_contiguous() and mix.dtype == torch.float32 and h.B == B and h.W == W, (mix.shape, h.B, h.W)
    assert w.is_contiguous() and tuple(w.shape) == (2, h.C)
    out = torch.empty((B, 2, out_bin, W - 2 * offset), device=mix.device, dtype=torch.float32)
    _call("evk_vr_mask_head", *h.args(), _p(w), h.C, _p(mix), _p(out), B, h.H, out_bin, W, offset, split_bin,
          ctypes.c_float(e_lo), ctypes.c_float(e_hi), 1 if use_agg else 0)
    return out


def transpose_rows(x, out=None):
    """[B, T, C] -> [B, C, T] (evk_transpose_rows): x contiguous fp32; `out` may be given as a contiguous [B, C, T]"""
    assert x.dim() == 3 and x.is_contiguous() and x.dtype == torch.float32 and x.is_cuda, (x.shape, x.dtype)
    B, T, C = x.shape
    if out is None:
        out = torch.empty((B, C, T), device=x.device, dtype=torch.float32)
    assert out.is_contiguous() and tuple(out.shape) == (B, C, T)
    _call("evk_transpose_rows", _p(x), C, T * C, _p(out), T, C * T, B, T, C, 0)
    return out


def lstm_bidir(g, w_hh, order="tn"):
    """Recurrence of a bidirectional one-layer nn.LSTM (evk_lstm_bidir_fwd).  g: the input projections with both biases
    added, [T, N, 8H] (order "tn") or [N, T, 8H] (order "nt"), last axis [direction][gate i, f, g, o][H]; w_hh [2, 4H, H].
    -> y with g's leading axes and 2H columns [h_forward | h_reverse], the nn.LSTM output layout."""
    assert g.dim() == 3 and g.is_contiguous() and g.dtype == torch.float32 and g.is_cuda, (g.shape, g.dtype)
    H = w_hh.shape[-1]
    assert w_hh.is_contiguous() and tuple(w_hh.shape) == (2, 4 * H, H) and g.shape[2] == 8 * H, (g.shape, w_hh.shape)
    T, N = g.shape[:2] if order == "tn" else g.shape[1::-1]
    y = torch.empty(g.shape[:2] + (2 * H,), device=g.device, dtype=torch.float32)
    gs, ys = (g.stride(0), g.stride(1)), (y.stride(0), y.stride(1))
    if order != "tn":
        gs, ys = gs[::-1], ys[::-1]
    _call_f("evk_lstm_bidir_fwd", 2.0 * 2 * T * N * 4 * H * H, _p(g), *gs, _p(w_hh), _p(y), *ys, T, N, H)
    return y


# ------------------------------------------------------------------------------------------------
# BS-Roformer and Mel-Band Roformer (bs_roformer.py, mel_band_roformer.py): rotary gated attention, band input, row norm,
# averaged band masks, inverse STFT
# ------------------------------------------------------------------------------------------------
def linear_into(x, w: PackedW, y, bias=None, act=ACT_NONE, res=None):
    """y = act(x W^T + bias + res) written into y (no autograd): x [rows, C] and y [rows, N] are 2-D views with unit column
    stride and any row pitch (column slices of wider buffers), res [rows, N] contiguous or None."""
    rows, C = x.shape
    N = w.D0
    assert w.Q == 1 and y.shape == (rows, N) and C <= w.pa.shape[2], (x.shape, y.shape, w.pa.shape)
    _fwd_like(x.unsqueeze(0), rows, w.pa, w.pa.shape[2], N * w.pa.shape[2], C, N, y.unsqueeze(0), J=rows, P=1, is_=1, off=[0],
              bias=bias, res=res.unsqueeze(0) if res is not None else None, act=act)
    return y


# ---- 16-bit Linears (linear_h16.cu): h(x) . h(W) on fp16 / bf16 tensor cores with fp32 accumulation ------------------
H16_TYPES = (torch.float16, torch.bfloat16)


class PackedH16:
    """A Linear's weight for the 16-bit kernels: w [N, ldw] fp16 or bf16, ldw = K rounded up to 64, zero past column K."""
    __slots__ = ("w", "K")

    def __init__(self, w, K):
        self.w, self.K = w, K


def pack_weight_h16(w, dtype):
    """nn.Linear weight [N, K] -> PackedH16 rounded to `dtype` (torch.float16 or torch.bfloat16) to nearest even, in the
    layout evk_linear_h16 and evk_linear_rows_h16 read.  A weight that is already exactly 16-bit keeps its bits."""
    if dtype not in H16_TYPES:
        raise ValueError(f"16-bit compute type {dtype} (torch.float16 or torch.bfloat16)")
    N, K = w.shape
    p = torch.zeros(N, (K + 63) // 64 * 64, dtype=dtype, device=w.device)
    p[:, :K] = w.detach()
    return PackedH16(p, K)


def _linear_h16(name, x, w: PackedH16, bias, act, res, out):
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    if x2.stride(1) != 1:
        x2 = x2.contiguous()
    rows, N = x2.shape[0], w.w.shape[0]
    assert K == w.K and x2.dtype == torch.float32 and rows >= 1, (x.shape, w.K, x2.dtype)
    y = torch.empty(x.shape[:-1] + (N,), device=x.device, dtype=torch.float32) if out is None else out
    y2 = y.reshape(-1, N) if out is None else out
    assert y2.shape == (rows, N) and y2.stride(1) == 1, (y2.shape, y2.stride())
    r2 = None
    if res is not None:
        r2 = res.reshape(rows, N)
        assert r2.stride(1) == 1, r2.stride()
    _call_f(name, 2.0 * rows * N * K, _p(x2), x2.stride(0), rows, _p(w.w), w.w.shape[1], int(w.w.dtype == torch.bfloat16),
            _p(bias), _p(r2), r2.stride(0) if r2 is not None else 0, _p(y2), y2.stride(0), N, K, int(act), ctypes.c_float(0.0))
    return y


def linear_h16(x, w: PackedH16, bias=None, act=ACT_NONE, res=None, out=None):
    """act(h(x) h(W)^T + bias + res) for many rows (evk_linear_h16: the 16-bit wgmma kernel).  x [..., K] fp32 with unit
    column stride; res shaped like the output; out: a [rows, N] view with unit column stride to write into (column slices of
    wider buffers), or None.  No gradient."""
    return _linear_h16("evk_linear_h16", x, w, bias, act, res, out)


def linear_rows_h16(x, w: PackedH16, bias=None, act=ACT_NONE, res=None, out=None):
    """linear_h16 for the few rows of a decode step (evk_linear_rows_h16): any row count, and a row's bits do not depend on
    how many rows share the launch."""
    return _linear_h16("evk_linear_rows_h16", x, w, bias, act, res, out)


def rope_attn(qkvg, cs, out, heads, L, n_outer, s_outer, n_inner, s_inner, s_tok):
    """evk_rope_attn_fwd: qkvg [rows, ld] token rows [q | k | v | gate logits], cs [L, 32, 2] (cos, sin) -> out [rows, heads*64];
    sequence (u, w) holds rows u*s_outer + w*s_inner + t*s_tok, t < L."""
    assert qkvg.dim() == 2 and qkvg.stride(1) == 1 and out.dim() == 2 and out.stride(1) == 1 and cs.is_contiguous()
    assert cs.shape[0] >= L
    _call_f("evk_rope_attn_fwd", 4.0 * n_outer * n_inner * heads * L * L * 64, _p(qkvg), qkvg.stride(0), _p(cs), _p(out),
            out.stride(0), heads, L, n_outer, s_outer, n_inner, s_inner, s_tok)
    return out


def rope_attn_h16(qkvg, cs, out, heads, L, n_outer, s_outer, n_inner, s_inner, s_tok, dtype):
    """rope_attn with 16-bit operands (evk_rope_attn_fwd_h16): rotated q, k, v and the probabilities rounded to `dtype`
    (torch.float16 or torch.bfloat16), fp32 accumulation, softmax and gate."""
    if dtype not in H16_TYPES:
        raise ValueError(f"16-bit compute type {dtype} (torch.float16 or torch.bfloat16)")
    assert qkvg.dim() == 2 and qkvg.stride(1) == 1 and out.dim() == 2 and out.stride(1) == 1 and cs.is_contiguous()
    assert cs.shape[0] >= L
    _call_f("evk_rope_attn_fwd_h16", 4.0 * n_outer * n_inner * heads * L * L * 64, _p(qkvg), qkvg.stride(0), _p(cs), _p(out),
            out.stride(0), heads, L, n_outer, s_outer, n_inner, s_inner, s_tok, int(dtype == torch.bfloat16))
    return out


def row_norm(x, gamma=None, out=None):
    """x / max(||x||_2, 1e-12) per row of a [rows, C] view, times sqrt(C) * gamma when gamma is given (evk_row_norm); out may
    be x"""
    rows, C = x.shape
    assert x.stride(1) == 1
    assert gamma is None or (gamma.is_contiguous() and gamma.numel() == C and gamma.dtype == torch.float32)
    out = torch.empty((rows, C), device=x.device, dtype=torch.float32) if out is None else out
    _call("evk_row_norm", _p(x), x.stride(0), _p(gamma), _p(out), out.stride(0), rows, C)
    return out


def band_input(cplx, B, S, band_off, bins, out):
    """evk_band_input: cplx [B*S, T, n_bins, 2] (ops.stft) -> out [B*T, >= 2*S*len(bins)]: band i's bins
    bins[band_off[i]:band_off[i+1]] in 'b t (f s c)' order, each band's segment L2-normalised; band_off, bins int32 device
    (BS-Roformer's bins: arange(n_bins))."""
    _, T, nb, _ = cplx.shape
    assert cplx.is_contiguous() and out.stride(1) == 1 and band_off.dtype == torch.int32 and bins.dtype == torch.int32
    assert out.shape[0] == B * T and out.shape[1] >= 2 * S * bins.numel()
    _call("evk_band_input", _p(cplx), B, S, T, nb, _p(band_off), _p(bins), band_off.numel() - 1, _p(out), out.stride(0))
    return out


def melband_mask_avg(g, S, cover_off, cover, out):
    """evk_melband_mask_avg: band-major complex masks g [rows, 2*S*n_slots] -> out [rows, 2*S*n_bins] (evk_istft's mask
    layout), each (bin, channel) the mean over the bands covering the bin; cover_off int32 device [n_bins + 1], cover int32
    device: the slots of each bin in ascending band order."""
    rows = g.shape[0]
    n_bins = cover_off.numel() - 1
    assert g.stride(1) == 1 and out.stride(1) == 1 and out.shape == (rows, 2 * S * n_bins)
    assert cover_off.dtype == torch.int32 and cover.dtype == torch.int32
    _call("evk_melband_mask_avg", _p(g), g.stride(0), _p(cover_off), _p(cover), S, n_bins, rows, _p(out), out.stride(0))
    return out


def istft(cplx, B, S, n_fft, hop, mask=None, out=None, work=None, length=None):
    """torch.istft(center=True, Hann(n_fft)) of cplx [B*S, T, n_fft/2+1, 2] (times the complex mask [B*T, (f s c)] when given)
    -> [B*S, hop*(T-1)], or [B*S, length] as torch.istft(length=length) (evk_istft).  work: scratch of B*S*T*n_fft floats
    (allocated when None)."""
    T = cplx.shape[1]
    assert cplx.is_contiguous() and cplx.shape[2] == n_fft // 2 + 1
    if out is None:
        out = torch.empty((B * S, hop * (T - 1) if length is None else length), device=cplx.device, dtype=torch.float32)
    if work is None:
        work = torch.empty(B * S * T * n_fft, device=cplx.device, dtype=torch.float32)
    assert work.numel() >= B * S * T * n_fft and out.stride(1) == 1
    if mask is not None:
        assert mask.stride(1) == 1 and mask.shape[0] == B * T
    ldm = mask.stride(0) if mask is not None else 0
    _call("evk_istft", _p(cplx), _p(mask), ldm, B, S, T, n_fft, hop, 0 if length is None else int(length), _p(work), _p(out),
          out.stride(0))
    return out


def vr_band_stft(wav, bands, l, row_gain, n_rows, high_band=-1, high_lo=0, high_h=0, zero_pad=True):
    """evk_vr_band_stft: wav a flat fp32 device buffer holding every band's two rows; bands: one (offset, L, ldw, n_fft, hop,
    crop_start, crop_stop, row0) tuple per band -> (combined spectrogram [2, n_rows, l, 2] (re, im; rows no band covers are
    zero), the high-end slice [2, high_h, l, 2] of band high_band or None)"""
    spec = torch.zeros((2, n_rows, l, 2), device=wav.device, dtype=torch.float32)
    high = torch.empty((2, high_h, l, 2), device=wav.device, dtype=torch.float32) if high_band >= 0 else None
    desc = (ctypes.c_int64 * (8 * len(bands)))(*[int(v) for b in bands for v in b])
    assert wav.is_contiguous() and row_gain.numel() == n_rows
    _call("evk_vr_band_stft", _p(wav), desc, len(bands), l, _p(row_gain), _p(spec), n_rows, high_band, high_lo, high_h, _p(high),
          1 if zero_pad else 0)
    return spec, high


def vr_mag_norm(spec):
    """evk_vr_mag_norm: complex spec [..., 2] -> (|spec| / max|spec| [...], max|spec| as a device tensor [1])"""
    assert spec.is_contiguous() and spec.shape[-1] == 2
    mag = torch.empty(spec.shape[:-1], device=spec.device, dtype=torch.float32)
    coef = torch.empty(1, device=spec.device, dtype=torch.float32)
    _call("evk_vr_mag_norm", _p(spec), mag.numel(), _p(mag), _p(coef))
    return mag, coef


def resample_poly(x, h, up, down, n_pre_remove, n_out, out=None):
    """evk_resample_poly: scipy.signal.resample_poly of the rows of x [rows, L] with the zero-prefixed fp32 filter h (device)
    -> [rows, n_out]"""
    rows, L = x.shape
    assert x.stride(1) == 1 and h.is_contiguous()
    out = torch.empty((rows, n_out), device=x.device, dtype=torch.float32) if out is None else out
    assert out.stride(1) == 1 and out.shape == (rows, n_out)
    _call("evk_resample_poly", _p(x), rows, L, x.stride(0), _p(h), h.numel(), up, down, n_pre_remove, _p(out), n_out, out.stride(0))
    return out


def ssl_normalize(a, lens):
    """evk_ssl_normalize: Normalize._name2go's loudness normalisation of the rows of a [B, L] (fp32 device, row b holding
    lens[b] samples; lens int32 device [B]) -> (a32 int16 [B, L], a32b fp32 [B, L], status int32 [B]: EVK_SSL_OK = 0,
    EVK_SSL_SKIP = 1, EVK_SSL_NONFINITE = 2); entries past a row's length are 0."""
    assert a.dim() == 2 and a.dtype == torch.float32 and a.stride(1) == 1
    assert lens.dtype == torch.int32 and lens.is_cuda and lens.numel() == a.shape[0]
    B, L = a.shape
    a32 = torch.empty((B, L), device=a.device, dtype=torch.int16)
    a32b = torch.empty((B, L), device=a.device, dtype=torch.float32)
    status = torch.empty(B, device=a.device, dtype=torch.int32)
    _call("evk_ssl_normalize", _p(a), a.stride(0), _p(lens.contiguous()), B, L, _p(a32), L, _p(a32b), L, _p(status))
    return a32, a32b, status


def frame_rms(x, lens, win, hop):
    """evk_frame_rms: Slicer.get_rms of the rows of x [B, L] (fp32 device, row b holding lens[b] samples; lens int32 device
    [B]) -> rms fp32 [B, 1 + (L + 2 (win // 2) - win) // hop]; frames past a row's own count are 0."""
    assert x.dim() == 2 and x.dtype == torch.float32 and x.is_cuda and x.stride(1) == 1
    assert lens.dtype == torch.int32 and lens.is_cuda and lens.numel() == x.shape[0]
    B, Lm = x.shape
    T = 1 + (Lm + 2 * (win // 2) - win) // hop
    assert T >= 1, (Lm, win, hop)
    rms = torch.empty((B, T), device=x.device, dtype=torch.float32)
    _call("evk_frame_rms", _p(x), x.stride(0), _p(lens.contiguous()), B, win, hop, _p(rms), T, T)
    return rms


SLICE_MAX_CHUNKS = 65535        # chunks of one evk_slice_normalize call


def slice_normalize(x, chunks, max_len, c1, c2, out=None):
    """evk_slice_normalize: the chunk loop of AudioService.slicer over the flat fp32 device buffer x.  chunks: int64 device
    [n, 2] = (offset, length), max_len >= every length -> (int16 buffer shaped like x, written at the chunks' offsets only,
    m fp32 [n] = max |chunk|, status int32 [n]: EVK_SLICE_OK = 0, EVK_SLICE_SILENT = 1, EVK_SLICE_NONFINITE = 2)."""
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    assert chunks.dtype == torch.int64 and chunks.is_cuda and chunks.is_contiguous() and chunks.dim() == 2 and chunks.shape[1] == 2
    n = chunks.shape[0]
    out = torch.empty(x.shape, device=x.device, dtype=torch.int16) if out is None else out
    assert out.dtype == torch.int16 and out.is_contiguous() and out.shape == x.shape
    m = torch.empty(n, device=x.device, dtype=torch.float32)
    status = torch.empty(n, device=x.device, dtype=torch.int32)
    for i in range(0, n, SLICE_MAX_CHUNKS):
        k = min(SLICE_MAX_CHUNKS, n - i)
        _call("evk_slice_normalize", _p(x), _p(chunks[i:]), k, int(max_len), float(c1), float(c2), _p(out), _p(m[i:]), _p(status[i:]))
    return out, m, status


def fragment_int16(x, frags, dst, max_len, gap, out):
    """evk_fragment_int16: TTS.audio_postprocess over the flat fp32 device buffer x.  frags: int64 device [n, 2] = (offset in x,
    length), dst: int64 device [n] = offset in out, max_len >= every length, gap the zero samples after every fragment; out:
    int16 device buffer, written at [dst, dst + length + gap) of every fragment.  -> m fp32 [n] = max |fragment|."""
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    assert frags.dtype == torch.int64 and frags.is_cuda and frags.is_contiguous() and frags.dim() == 2 and frags.shape[1] == 2
    assert dst.dtype == torch.int64 and dst.is_contiguous() and dst.shape == (frags.shape[0],)
    assert out.dtype == torch.int16 and out.is_cuda and out.is_contiguous()
    n = frags.shape[0]
    m = torch.empty(n, device=x.device, dtype=torch.float32)
    for i in range(0, n, SLICE_MAX_CHUNKS):
        k = min(SLICE_MAX_CHUNKS, n - i)
        _call("evk_fragment_int16", _p(x), _p(frags[i:]), _p(dst[i:]), k, int(max_len), int(gap), _p(out), _p(m[i:]))
    return m


def vr_assemble(x, pred, pred_tta, coef, bands, gains, high=None, mirror_lo=0, top=-1):
    """evk_vr_assemble: combined spectrogram x [2, n_rows, l, 2], pred / pred_tta [2, n_rows, l] and coef [1] -> one
    [4, l, n_fft/2+1, 2] frame tensor per band (rows y ch0, y ch1, v ch0, v ch1: evk_istft's input with B = 4, S = 1).
    bands: (n_fft, crop_start, crop_stop, row0) per band; gains: one fp32 device vector of n_fft/2+1 per band."""
    _, n_rows, l, _ = x.shape
    assert x.is_contiguous() and pred.is_contiguous() and (pred_tta is None or pred_tta.is_contiguous())
    nbs = [b[0] // 2 + 1 for b in bands]
    out = torch.empty(sum(4 * l * nb * 2 for nb in nbs), device=x.device, dtype=torch.float32)
    g = torch.cat(gains).contiguous()
    desc, go, oo = [], 0, 0
    for b, nb in zip(bands, nbs):
        desc += [*b, go, oo]
        go, oo = go + nb, oo + 4 * l * nb
    high_h = high.shape[1] if high is not None else 0
    _call("evk_vr_assemble", _p(x), _p(pred), _p(pred_tta), _p(coef), n_rows, l, _p(high), high_h, mirror_lo, top,
          (ctypes.c_int64 * len(desc))(*desc), len(bands), _p(g), _p(out))
    frames, o = [], 0
    for nb in nbs:
        frames.append(out[o:o + 8 * l * nb].view(4, l, nb, 2))
        o += 8 * l * nb
    return frames


def glu_into(h, out):
    """nn.GLU(dim=-1) of h [rows, 2C] written into out [rows, C] (a view with unit column stride; evk_glu_res with x = NULL)"""
    rows, C2 = h.shape
    assert h.stride(1) == 1 and out.stride(1) == 1 and out.shape == (rows, C2 // 2)
    _call("evk_glu_res", None, 0, _p(h), h.stride(0), _p(out), out.stride(0), rows, C2 // 2)
    return out


# ------------------------------------------------------------------------------------------------
# MDX23C (mdx23c.py): plane instance norm, TDF Linear, transposed 2x2 conv, spectral layouts, residual adds
# ------------------------------------------------------------------------------------------------
C2_GELU = 4


def instnorm_plane(x: CLView, gamma, beta, y: CLView, eps=1e-5, gelu_after=True):
    """nn.InstanceNorm2d(affine=True) over the H*W pixels of each (item, channel) of x (+ exact GELU) into y
    (evk_instnorm_plane); x and y cover whole [B, H, W] planes, each a channel slice of its buffer."""
    assert x.r0 == 0 and x.H == x.buf.shape[1] and (y.B, y.H, y.W, y.C) == (x.B, x.H, x.W, x.C)
    assert gamma.is_contiguous() and beta.is_contiguous() and gamma.numel() == x.C and beta.numel() == x.C
    _call("evk_instnorm_plane", x.args()[0], x.args()[1], _p(gamma), _p(beta), ctypes.c_float(eps), 1 if gelu_after else 0,
          y.args()[0], y.args()[1], x.B, x.H * x.W, x.C)
    return y


def mdx_tdf(x: CLView, w, y: CLView, res: CLView = None):
    """y[b, h, m, :] = sum_k w[m, k] x[b, h, k, :] (+ res) along the frequency (W) axis (evk_mdx_tdf): w [W_out, W_in]"""
    M, K = w.shape
    assert w.is_contiguous() and x.W == K and (y.B, y.H, y.W, y.C) == (x.B, x.H, M, x.C), (w.shape, x.W, y.W)
    (xp, xl, _), (yp, yl, _) = x.args(), y.args()
    r = res.args() if res is not None else (None, 0, 0)
    if res is not None:
        assert (res.B, res.H, res.W, res.C) == (y.B, y.H, y.W, y.C)
    _call_f("evk_mdx_tdf", 2.0 * x.B * x.H * M * K * x.C, _p(w), xp, xl, K * xl, r[0], r[1],
            M * r[1], yp, yl, M * yl, x.B * x.H, M, x.C, K)
    return y


def convt2x2(x: CLView, w, y: CLView):
    """ConvTranspose2d(kernel 2, stride 2, no bias) (evk_convt2x2_fwd): w [2, 2, N, C]; y [B, 2H, 2W, N]"""
    N = w.shape[2]
    assert w.is_contiguous() and tuple(w.shape) == (2, 2, N, x.C) and (y.B, y.H, y.W, y.C) == (x.B, 2 * x.H, 2 * x.W, N)
    assert x.r0 == 0 and y.r0 == 0 and x.H == x.buf.shape[1] and y.H == y.buf.shape[1]
    _call_f("evk_convt2x2_fwd", 2.0 * x.B * x.H * x.W * 4 * N * x.C, *x.args(), _p(w), *y.args(), x.B, x.H, x.W, x.C, N)
    return y


def mdx_front(cplx, B, S, k, F, y: CLView):
    """evk_mdx_front: cplx [B*S, T, n_bins, 2] (ops.stft) -> y [B, T, F, 2*S*k] (cac2cws of the first k*F bins)"""
    _, T, nb, _ = cplx.shape
    assert cplx.is_contiguous() and y.r0 == 0 and (y.B, y.H, y.W, y.C) == (B, T, F, 2 * S * k)
    _call("evk_mdx_front", _p(cplx), B, S, T, nb, k, F, y.args()[0], y.args()[1])
    return y


def mdx_back(x: CLView, nt, S, k, n_bins, out=None):
    """evk_mdx_back: x [B, T, F, nt*2*S*k] -> cplx [B*nt*S, T, n_bins, 2] (cws2cac, zero bins from k*F on)"""
    B, T, F = x.B, x.H, x.W
    assert x.r0 == 0 and x.C == nt * 2 * S * k
    out = torch.empty((B * nt * S, T, n_bins, 2), device=x.buf.device, dtype=torch.float32) if out is None else out
    assert out.is_contiguous() and tuple(out.shape) == (B * nt * S, T, n_bins, 2)
    _call("evk_mdx_back", x.args()[0], x.args()[1], B, nt, S, T, n_bins, k, F, _p(out))
    return out


def mdx_add(a: CLView, b: CLView, y: CLView, m: CLView = None):
    """y = (a + b) * m (evk_mdx_add; m optional) over whole planes of equal shape"""
    for v in (a, b, y) + ((m,) if m is not None else ()):
        assert v.r0 == 0 and v.H == v.buf.shape[1] and (v.B, v.H, v.W, v.C) == (a.B, a.H, a.W, a.C)
    ma = m.args() if m is not None else (None, 0, 0)
    _call("evk_mdx_add", a.args()[0], a.args()[1], b.args()[0], b.args()[1], ma[0], ma[1], y.args()[0], y.args()[1],
          a.B * a.H * a.W, a.C)
    return y


# ------------------------------------------------------------------------------------------------
# Whisper transcription (whisper.py): log-mel front end, decode attention with slot tables, beam step
# ------------------------------------------------------------------------------------------------
def whisper_logmel(wav, lens, T, basis, fb):
    """evk_whisper_logmel: wav [B, L] fp32 (row b holds lens[b] 16 kHz samples; lens int32 device [B], lens[b] // 160 <= T),
    basis [2, 400, 201], fb [201, n_mels] -> [B, T, n_mels] normalised log-mel of each whole clip (max over all its frames),
    zero after its lens[b] // 160 frames.  T = 3000: the encoder's 30 s input."""
    assert wav.dim() == 2 and wav.stride(1) == 1 and lens.dtype == torch.int32 and basis.is_contiguous() and fb.is_contiguous()
    B, M = wav.shape[0], fb.shape[1]
    out = torch.empty((B, T, M), device=wav.device, dtype=torch.float32)
    part = torch.empty((B, (T + 255) // 256), device=wav.device, dtype=torch.float32)
    _call("evk_whisper_logmel", _p(wav), wav.stride(0), _p(lens), B, T, _p(basis), _p(fb), M, _p(part), _p(out))
    return out


def whisper_embed(tok, emb, pe, pos, out):
    """out[r] = emb[tok[r]] + pe[*pos] (evk_whisper_embed)."""
    _call("evk_whisper_embed", _p(tok), _p(emb), _p(pe), _p(pos), tok.numel(), emb.shape[1], _p(out))
    return out


def whisper_add_pos(x, pe):
    """x [B, T, d] (contiguous) += pe[:T] in place (evk_whisper_add_pos)."""
    assert x.is_contiguous() and pe.is_contiguous()
    B, T, d = x.shape
    _call("evk_whisper_add_pos", _p(x), B * T, T, d, _p(pe))
    return x


def whisper_self_kv(qkv, pool, tab, pos, S):
    """Write every row's K | V (columns d..3d of qkv [R, 3d]) into its slot r * S + *pos of pool [R * S, >= 2d] and list the
    slot in tab [R, >= S] (evk_whisper_self_kv)."""
    R, d = qkv.shape[0], qkv.shape[1] // 3
    assert qkv.stride(1) == 1 and pool.stride(1) == 1 and tab.dtype == torch.int32 and tab.stride(1) == 1
    _call("evk_whisper_self_kv", _p(qkv), qkv.stride(0), d, _p(pool), pool.stride(0), _p(tab), tab.stride(0), _p(pos), R, S)


def whisper_attn(q, kv, v_off, heads, out, *, tab=None, pos=None, n_keys, nq=1):
    """evk_whisper_attn, head dim 64, exact fp32.  tab given: row r attends the pool rows tab[r, :*pos + 1] (n_keys = table
    width); otherwise rows g * nq + a attend kv rows g * n_keys .. g * n_keys + n_keys - 1 (cross-attention of a clip's beams)."""
    assert q.stride(1) == 1 and kv.stride(1) == 1 and out.stride(1) == 1
    groups = q.shape[0] // nq
    _call_f("evk_whisper_attn", 4.0 * q.shape[0] * heads * n_keys * 64, _p(q), q.stride(0), _p(kv), kv.stride(0), v_off, _p(tab),
            tab.stride(0) if tab is not None else 0, _p(pos), n_keys, groups, nq, heads, ctypes.c_float(0.125), _p(out), out.stride(0))
    return out


def whisper_layernorm(x, gamma, beta, eps=1e-5):
    """evk_whisper_layernorm over the last dim of x (any width) -> a new tensor of x's shape."""
    x = _cl(x.detach())
    rows, C, ld = _rows(x)
    y = torch.empty(x.shape, device=x.device, dtype=torch.float32)
    _call("evk_whisper_layernorm", _p(x), ld, _p(gamma.detach()), _p(beta.detach()), ctypes.c_float(eps), _p(y), C, rows, C)
    return y


def whisper_first_pass(logits, nospeech, lang_ids, nsp, lang_tok):
    """evk_whisper_first_pass: nsp[r] = softmax(logits[r])[nospeech], lang_tok[r] = argmax of logits[r] over lang_ids."""
    assert logits.stride(1) == 1 and lang_ids.dtype == torch.int32
    _call("evk_whisper_first_pass", _p(logits), logits.stride(0), logits.shape[0], logits.shape[1], int(nospeech), _p(lang_ids),
          lang_ids.numel(), _p(nsp), _p(lang_tok))


def whisper_beam_step(logits, st, beam, lay, length_penalty=1.0, track_lse=False):
    """evk_whisper_beam_step on the decode state `st` (whisper.WhisperModel._state) with token layout `lay` =
    (eot, notimestamps, ts_begin, max_init_ts, prompt_len, max_length).  track_lse: also carry st["run_lse"] / st["fin_lse"],
    each hypothesis' sum of its processed rows' log-sum-exp (st["row_lse"] is scratch)."""
    clips = logits.shape[0] // beam
    assert st["fin_seq"].stride(1) == st["hist"].stride(0) and st["tab"].stride(0) <= 448
    lse = [_p(st[k]) if track_lse else None for k in ("row_lse", "run_lse", "fin_lse")]
    _call("evk_whisper_beam_step", _p(logits), logits.stride(0), clips, beam, logits.shape[1], *[int(v) for v in lay],
          _p(st["sup"]), st["sup"].numel(), _p(st["bsup"]), st["bsup"].numel(), _p(st["g"]), ctypes.c_float(length_penalty),
          _p(st["cv"]), _p(st["ci"]), _p(st["score"]), _p(st["hist"]), st["hist"].stride(0), _p(st["tab"]), st["tab"].stride(0),
          _p(st["tok"]), _p(st["parent"]), _p(st["fin_score"]), _p(st["fin_seq"]), _p(st["fin_len"]),
          _p(st["fin_flag"]), _p(st["unsat"]), *lse)


def whisper_window(lm, tab, out=None):
    """evk_whisper_window: lm [B, T, n_mels], tab int32 device [R, 3] of (clip, seek, n) -> [R, 3000, n_mels], row r the frames
    [seek, seek + n) of clip, zero after n."""
    assert lm.is_contiguous() and tab.dtype == torch.int32 and tab.is_contiguous() and tab.shape[1] == 3
    B, T, M = lm.shape
    R = tab.shape[0]
    out = torch.empty((R, 3000, M), device=lm.device, dtype=torch.float32) if out is None else out
    assert out.is_contiguous() and out.shape == (R, 3000, M)
    _call("evk_whisper_window", _p(lm), B, T, M, _p(tab), R, _p(out))
    return out
