"""One stage-2 (SoVITS + HiFi-GAN) optimisation step on the sm_90a kernels.

Mirrors /root/reference/src/train/sovits.py:459-525 (G forward, mel/slice features, D step, G step, two AdamW
updates) with these deliberate differences, none of which changes the math of the update:
  * fp32 storage / TF32 tensor-core math instead of fp16 autocast + GradScaler (no loss scaling needed);
  * the discriminators see real and generated audio as one 2B batch (models.py:606-612 runs them sequentially);
  * the G step does not compute (and all-reduce) discriminator weight gradients that the reference computes and
    then discards at the next ``optim_d.zero_grad()`` (SURVEY.md C1);
  * the grad-norm probe is one fused reduction inside the optimizer kernel instead of 883 ``.item()`` syncs
    (commons.py:140-155); nothing in the step synchronises with the host;
  * slice ids / posterior noise / dropout masks come from device-side Philox streams.
Data-parallel: gradients are summed across ranks with NCCL over one flat fp32 buffer per network, then the
1/world scaling is folded into the optimizer kernel.
"""
import math

import torch
import torch.distributed as dist

from .. import ops
from ..mel_processing import get_bank


class FlatAdamW:
    """AdamW (torch.optim.AdamW semantics, sovits.py:294-319) over per-group flat fp32 arenas.

    Parameters are re-pointed into one contiguous buffer per lr group, so the update is one kernel per group and the
    data-parallel all-reduce is one collective per network.

    `frozen` names parameters that never receive a gradient (the reference's `p.grad is None` case: torch.optim.AdamW
    skips them entirely -- no weight decay, no state).  They live in a tail region of the arena that no update kernel
    touches, keep their index in `param_groups` (so optimizer state indices line up with a torch.optim.AdamW built over
    the reference modules, whose named_parameters() order models.py reproduces) and have no entry in `state`."""

    def __init__(self, named_params, groups, betas, eps, weight_decay=0.01, frozen=()):
        # groups: list of (lr_scale, [names]) ; every param must appear exactly once
        self.betas, self.eps, self.wd = betas, eps, weight_decay
        named = dict(named_params)
        self.frozen = set(frozen)
        self.groups = []
        dev = next(iter(named.values())).device
        total = sum(named[n].numel() for _, names in groups for n in names)
        self.flat_p = torch.empty(total, device=dev, dtype=torch.float32)
        self.flat_g = torch.zeros(total, device=dev, dtype=torch.float32)
        off = 0
        self.slots = {}

        def place(n):
            nonlocal off
            p = named[n]
            k = p.numel()
            self.flat_p[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat_p[off:off + k].view_as(p)
            self.slots[n] = (off, k)
            off += k
        for lr_scale, names in groups:
            beg = off
            for n in names:
                if n not in self.frozen:
                    place(n)
            self.groups.append(dict(lr_scale=lr_scale, beg=beg, end=off, names=list(names)))
        self.n_active = off                                   # [0, n_active): updated + all-reduced; the rest is frozen
        for _, names in groups:
            for n in names:
                if n in self.frozen:
                    place(n)
        self.flat_m = torch.zeros(self.n_active, device=dev, dtype=torch.float32)
        self.flat_v = torch.zeros(self.n_active, device=dev, dtype=torch.float32)
        self.params = [named[n] for _, names in groups for n in names]
        self.names = [n for _, names in groups for n in names]
        self.hyper = torch.zeros(2, device=dev, dtype=torch.float32)        # [lr, step] lives on the device
        self.gnorm_sq = torch.zeros(1, device=dev, dtype=torch.float32)
        self.lr_host = 0.0

    @property
    def step_count(self):
        return int(self.hyper[1].item())

    @property
    def reduce_view(self):
        """what the data-parallel exchange sums: the gradients of the parameters that are actually updated"""
        return self.flat_g[:self.n_active]

    def set_lr(self, lr):
        """host-side (outside any captured graph): the lr only changes at epoch boundaries (ExponentialLR)."""
        self.lr_host = float(lr)
        self.hyper[0] = float(lr)

    def set_grads(self, grads):
        """copy autograd's per-parameter gradients into the flat buffer.  A parameter without a gradient must have been
        declared `frozen` (it is then skipped like torch.optim.AdamW skips `p.grad is None`); anything else is a bug."""
        views, srcs = [], []
        for n, g in zip(self.names, grads):
            off, k = self.slots[n]
            if g is None:
                if n not in self.frozen:
                    raise RuntimeError(f"parameter {n} received no gradient but is not declared frozen")
            elif n in self.frozen:
                raise RuntimeError(f"frozen parameter {n} received a gradient")
            else:
                views.append(self.flat_g[off:off + k].view_as(g))
                srcs.append(g)
        torch._foreach_copy_(views, srcs)

    def step(self, grad_scale=1.0):
        """graph-capturable: step counter, bias corrections and lr are read from device memory."""
        ops.scalar_add(self.hyper[1:], 1.0)
        self.gnorm_sq.zero_()
        for g in self.groups:
            s, e = g["beg"], g["end"]
            if e > s:
                ops.adamw_flat(self.flat_p[s:e], self.flat_g[s:e], self.flat_m[s:e], self.flat_v[s:e], self.hyper,
                               g["lr_scale"], self.betas, self.eps, self.wd, grad_scale, self.gnorm_sq)

    # torch.optim.AdamW-compatible state (ckpt.py:78-93 stores optimizer.state_dict(); the reference resumes from it with
    # torch.optim.AdamW.load_state_dict followed by ExponentialLR, which needs 'lr' / 'initial_lr' in every group)
    def state_dict(self):
        state = {}
        sc = self.step_count
        for i, n in enumerate(self.names):
            if n in self.frozen:
                continue
            off, k = self.slots[n]
            shape = self.params[i].shape
            state[i] = dict(step=torch.tensor(float(sc)), exp_avg=self.flat_m[off:off + k].view(shape).clone(),
                            exp_avg_sq=self.flat_v[off:off + k].view(shape).clone())
        pg, idx = [], 0
        for g in self.groups:
            n = len(g["names"])
            lr = self.lr_host * g["lr_scale"]
            pg.append(dict(lr=lr, betas=tuple(self.betas), eps=self.eps, weight_decay=self.wd, amsgrad=False, foreach=None,
                           maximize=False, capturable=False, differentiable=False, fused=None,
                           initial_lr=g.get("initial_lr", lr), params=list(range(idx, idx + n))))
            idx += n
        return dict(state=state, param_groups=pg)

    def load_state_dict(self, sd):
        """accepts this class's own checkpoints and torch.optim.AdamW's (same param order)."""
        groups = sd.get("param_groups", [])
        assert not groups or [len(g["params"]) for g in groups] == [len(g["names"]) for g in self.groups], \
            "optimizer state has a different parameter-group structure"
        for i, n in enumerate(self.names):
            st = sd["state"].get(i)
            if st is None or n in self.frozen:
                continue
            off, k = self.slots[n]
            self.flat_m[off:off + k].copy_(st["exp_avg"].reshape(-1))
            self.flat_v[off:off + k].copy_(st["exp_avg_sq"].reshape(-1))
            self.hyper[1] = float(st["step"])
        if groups and "lr" in groups[0]:
            self.set_lr(float(groups[0]["lr"]) / (self.groups[0]["lr_scale"] or 1.0))
            for mine, g in zip(self.groups, groups):
                if "initial_lr" in g:
                    mine["initial_lr"] = float(g["initial_lr"])


FROZEN_G = ("ssl_proj.weight", "ssl_proj.bias")     # models.py:911-921: the frozen quantizer's front end gets no gradient
CODEBOOK = tuple("quantizer.vq.layers.0._codebook." + n for n in ("embed", "embed_avg", "cluster_size", "inited"))


def g_param_groups(net_g, text_low_lr_rate):
    """sovits.py:286-312: text_embedding / encoder_text / mrte train at lr * text_low_lr_rate."""
    base, te, et, mr = [], [], [], []
    for n, _ in net_g.named_parameters():
        if n.startswith("enc_p.text_embedding."):
            te.append(n)
        elif n.startswith("enc_p.encoder_text."):
            et.append(n)
        elif n.startswith("enc_p.mrte."):
            mr.append(n)
        else:
            base.append(n)
    return [(1.0, base), (text_low_lr_rate, te), (text_low_lr_rate, et), (text_low_lr_rate, mr)]


def quantize_shape(T, X, t_q=32, x_q=32):
    """Pad targets for a batch whose longest item has T frames / X phonemes: CUDA graphs are captured per shape, so
    shapes are rounded up to a coarse grid (the length masks already make padding inert)."""
    return (T + t_q - 1) // t_q * t_q, (X + x_q - 1) // x_q * x_q


def pad_host_batch(host, Tq, Xq, hop):
    """zero-pad a collated host batch (data.TextAudioSpeakerCollate layout) to Tq frames / Xq phonemes."""
    B, _, T = host["ssl"].shape
    X = host["text"].shape[1]
    if T == Tq and X == Xq:
        return host
    assert Tq >= T and Xq >= X
    out = dict(host)
    F = torch.nn.functional
    out["ssl"] = F.pad(host["ssl"], (0, Tq - T))
    out["wav"] = F.pad(host["wav"], (0, Tq * hop - host["wav"].shape[2]))
    out["text"] = F.pad(host["text"], (0, Xq - X))
    return out


class S2Step:
    """Holds the two networks, both optimisers and runs `sovits.py:459-525` for one batch."""
    MAX_GRAPHS = 12          # LRU bound on captured shapes (all graphs share one memory pool)
    CAPTURE_AFTER = 2        # a shape is captured the 2nd time it is seen; rare shapes run the eager step

    def __init__(self, net_g, net_d, hps_train, hps_data, world_size=1):
        self.net_g, self.net_d = net_g, net_d
        self.t, self.d = hps_train, hps_data
        self.world = world_size
        self.seg_frames = hps_train["segment_size"] // hps_data["hop_length"]
        betas = tuple(hps_train["betas"])
        # freeze_quantizer: false trains ssl_proj and moves the codebook (an EMA of the batches' assignments)
        self.vq_train = net_g.freeze_quantizer is False
        self.opt_g = FlatAdamW(net_g.named_parameters(), g_param_groups(net_g, hps_train["text_low_lr_rate"]), betas,
                               hps_train["eps"], frozen=() if self.vq_train else FROZEN_G)
        self.opt_d = FlatAdamW(net_d.named_parameters(), [(1.0, [n for n, _ in net_d.named_parameters()])], betas,
                               hps_train["eps"])
        self.lr = hps_train["learning_rate"]
        self.opt_g.set_lr(self.lr)
        self.opt_d.set_lr(self.lr)
        dev = next(net_g.parameters()).device
        self.bank = get_bank(hps_data["sampling_rate"], hps_data["filter_length"], hps_data["n_mel_channels"],
                             hps_data["mel_fmin"], hps_data["mel_fmax"], dev)
        self._graphs = {}            # shape key -> (graphs, static inputs, static outputs); insertion order = LRU order
        self._seen = {}              # shape key -> sightings
        self._pool = None            # one private memory pool shared by every captured graph
        self._shape_group = None     # gloo group for the host-side shape agreement (world > 1)

    def losses(self, batch, noise=None, ids_slice=None, kmeans_idx=None):
        """Forward + both losses (no optimiser).  batch: dict of channels-last device tensors:
        ssl [B,T,768], spec [B,T,1025], lengths int32 [B], wav [B,L,1], text int64 [B,X], text_lengths int32 [B],
        optionally vq_rows int32 [1] (the trainable quantizer's reference row count, see SynthesizerTrn.forward_cl)."""
        hop, seg = self.d["hop_length"], self.t["segment_size"]
        r = self.net_g.forward_cl(batch["ssl"], batch["spec"], batch["lengths"], batch["text"], batch["text_lengths"],
                                  noise, ids_slice, batch.get("vq_rows"), kmeans_idx)
        ids = r["ids_slice"]
        y_hat = r["y_hat"]                                                        # [B, seg, 1]
        B = y_hat.shape[0]
        mel = ops.spec_to_mel(batch["spec"], self.bank)                            # sovits.py:470-477
        y_mel = ops.slice_rows(mel, ids, self.seg_frames)
        _, y_hat_mel = ops.mel_frontend(y_hat.reshape(B, seg), self.bank, hop)     # sovits.py:481-490
        y = ops.slice_rows(batch["wav"], ids, seg, mul=hop)                        # sovits.py:492-494
        r.update(y=y, y_mel=y_mel, y_hat_mel=y_hat_mel)
        return r

    def d_loss(self, r):
        B = r["y"].shape[0]
        outs = self.net_d.forward_cl(r["y"], r["y_hat"].detach())                  # sovits.py:497
        loss = 0
        for logit, _ in outs:
            loss = loss + ops.mean_sq_one_minus(logit[:B]) + ops.mean_sq(logit[B:])
        return loss

    def g_loss(self, r):
        B = r["y"].shape[0]
        outs = self.net_d.forward_cl(r["y"], r["y_hat"], weights_need_grad=False)  # sovits.py:511
        loss_mel = ops.mean_abs_diff(r["y_hat_mel"], r["y_mel"]) * self.t["c_mel"]
        loss_kl = ops.kl_loss(r["z_p"], r["logs_q"], r["m_p"], r["logs_p"], r["lengths"]) * self.t["c_kl"]
        loss_fm, loss_gen = 0, 0
        for logit, fmap in outs:
            for f in fmap:
                loss_fm = loss_fm + ops.mean_abs_diff(f[B:], f[:B])
            loss_gen = loss_gen + ops.mean_sq_one_minus(logit[B:])
        loss_fm = loss_fm * 2
        total = loss_gen + loss_fm + loss_mel + loss_kl                            # + kl_ssl == 0 (frozen quantizer)
        parts = dict(loss_gen=loss_gen, loss_fm=loss_fm, loss_mel=loss_mel, loss_kl=loss_kl)
        if "kl_ssl" in r:                                                          # sovits.py:518: + kl_ssl * 1
            total = total + r["kl_ssl"]
            parts["kl_ssl"] = r["kl_ssl"]
        c_mr = float(self.t.get("c_mrstft", 0.0))
        if c_mr > 0.0:          # opt-in extension (BASELINE config 5): the MR-STFT term of bs_roformer.py:565-581 on the fused STFT kernel
            parts["loss_mrstft"] = ops.mrstft_loss(r["y_hat"].reshape(B, -1), r["y"].reshape(B, -1)) * c_mr
            total = total + parts["loss_mrstft"]
        return total, parts

    def _allreduce(self, opt):
        if self.world > 1:
            dist.all_reduce(opt.reduce_view)

    def _broadcast_codebook(self):
        """DDP(broadcast_buffers=True) semantics of the reference (sovits.py:321): before every G forward rank 0's codebook
        buffers replace every other rank's, so codes come from rank 0's codebook and only rank 0's EMA survives."""
        if self.vq_train and self.world > 1:
            for n in CODEBOOK:
                dist.broadcast(self.net_g.P(n), src=0)

    # The step in three segments, split where the data-parallel gradient exchanges happen:
    #   A: G forward, features, D forward, D backward -> flat D grads          | all-reduce(D grads)
    #   B: D AdamW, D forward (updated weights), G backward -> flat G grads    | all-reduce(G grads)
    #   C: G AdamW, RNG advance
    # EVK_NVTX=1 brackets the phases with NVTX ranges (ncu --nvtx --nvtx-include "s2/d_backward/" ... selects a phase's kernels).
    def _seg_a(self, batch, noise=None, ids_slice=None, kmeans_idx=None):
        with ops.nvtx_range("s2/forward"):
            r = self.losses(batch, noise, ids_slice, kmeans_idx)
            loss_d = self.d_loss(r)
        with ops.nvtx_range("s2/d_backward"), ops.grad_pool():
            self.opt_d.set_grads(torch.autograd.grad(loss_d, self.opt_d.params, allow_unused=True))
        return r, loss_d

    def _seg_b(self, r):
        with ops.nvtx_range("s2/d_adamw"):
            self.opt_d.step(1.0 / self.world)
        with ops.nvtx_range("s2/g_loss_forward"):
            loss_g, parts = self.g_loss(r)
        with ops.nvtx_range("s2/g_backward"), ops.grad_pool():
            self.opt_g.set_grads(torch.autograd.grad(loss_g, self.opt_g.params, allow_unused=True))
        return loss_g, parts

    def _seg_c(self):
        with ops.nvtx_range("s2/g_adamw"):
            self.opt_g.step(1.0 / self.world)
            ops.advance_rng()

    @staticmethod
    def _outputs(loss_d, loss_g, parts, opt_d, opt_g):
        out = dict(loss_disc=loss_d.detach(), loss_gen_all=loss_g.detach(), grad_norm_d=opt_d.gnorm_sq, grad_norm_g=opt_g.gnorm_sq)
        out.update({k: v.detach() for k, v in parts.items()})
        return out

    def step(self, batch, noise=None, ids_slice=None, collectives=True, kmeans_idx=None):
        """Eager step (every kernel launched from Python).  No host synchronisation anywhere, except that a trainable
        quantizer reads its `inited` flag once.  collectives=False runs the rank-local math only (graph warm-up: a warm-up
        must never pair with another rank's real gradient exchange).  kmeans_idx: see SynthesizerTrn.forward_cl."""
        if collectives:
            self._broadcast_codebook()
        r, loss_d = self._seg_a(batch, noise, ids_slice, kmeans_idx)
        if collectives:
            self._allreduce(self.opt_d)
        loss_g, parts = self._seg_b(r)
        if collectives:
            self._allreduce(self.opt_g)
        self._seg_c()
        return self._outputs(loss_d, loss_g, parts, self.opt_d, self.opt_g)

    # ---- shape agreement + CUDA-graph path ----------------------------------------------------------------------
    def agree_shape(self, T, X):
        """-> (Tq, Xq): the padded shape EVERY rank uses for this iteration.  Each rank's collate pads to its own batch
        maximum (data_utils.py:185-188), so the local maxima are first rounded up to a coarse grid and then MAX-reduced
        over a gloo (host-side) group: no GPU synchronisation, and all ranks capture / replay / fall back to the eager
        step at the same iterations, so their NCCL all-reduces always pair up."""
        Tq, Xq = quantize_shape(T, X)
        if self.world > 1:
            if self._shape_group is None:
                self._shape_group = dist.new_group(backend="gloo")
            t = torch.tensor([Tq, Xq], dtype=torch.int64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self._shape_group)
            Tq, Xq = int(t[0]), int(t[1])
        return Tq, Xq

    def train_step(self, batch):
        """What the trainer calls: replay the graph of this (already agreed / quantised) shape, capturing it the
        CAPTURE_AFTER-th time the shape shows up; before that the eager step runs."""
        key = (tuple(batch["ssl"].shape), tuple(batch["text"].shape))
        n = self._seen[key] = self._seen.get(key, 0) + 1
        if self.vq_train and self.net_g.codebook_needs_init():
            return self.step(batch)              # the k-means initialisation runs once, eagerly
        if key in self._graphs or n >= self.CAPTURE_AFTER:
            return self.graph_step(batch)
        return self.step(batch)

    def graph_step(self, batch, noise=None, ids_slice=None, keep=False):
        """Copy `batch` into the static input buffers of the graph captured for its shape, replay, return the static
        loss tensors.  noise / ids_slice (parity tests) become static inputs of a separately keyed graph; keep=True also
        returns the captured forward tensors (they stay valid until the next replay)."""
        key = (tuple(batch["ssl"].shape), tuple(batch["text"].shape), noise is not None, bool(keep))
        if self.vq_train and self.net_g.codebook_needs_init():
            raise RuntimeError("the codebook is not initialised yet (inited == 0): run one eager step() first")
        g = self._graphs.pop(key, None)
        if g is None:
            while len(self._graphs) >= self.MAX_GRAPHS:                  # evict the least recently used shape
                self._graphs.pop(next(iter(self._graphs)))
            inputs = dict(batch)
            if noise is not None:
                inputs["noise"], inputs["ids_slice"] = noise, ids_slice
            g = self._capture(inputs, keep)
        self._graphs[key] = g                                            # (re)insert as most recently used
        graphs, static, out = g
        for k in static:
            src = noise if k == "noise" else ids_slice if k == "ids_slice" else batch[k]
            if static[k] is not src:
                static[k].copy_(src, non_blocking=True)
        self._broadcast_codebook()
        if len(graphs) == 1:
            graphs[0].replay()
        else:                               # data parallel: NCCL all-reduces run between the captured segments
            graphs[0].replay()
            self._allreduce(self.opt_d)
            graphs[1].replay()
            self._allreduce(self.opt_g)
            graphs[2].replay()
        return out

    def _capture(self, batch, keep=False):
        static = {k: (v.clone() if k != "spec" else v) for k, v in batch.items()}
        # `spec` keeps its padded row pitch (a view of a wider buffer): clone the parent storage explicitly
        sp = batch["spec"]
        wide = torch.zeros((sp.shape[0], sp.shape[1], sp.stride(1)), device=sp.device, dtype=sp.dtype)   # pitch columns must stay zero (ops.widen_to_pitch)
        static["spec"] = wide[:, :, :sp.shape[2]]
        static["spec"].copy_(sp)
        inj = dict(noise=static.get("noise"), ids_slice=static.get("ids_slice"))
        feed = {k: v for k, v in static.items() if k not in ("noise", "ids_slice")}
        # warm-up (allocator, smem attributes) must not count as training: snapshot and restore all mutable state.
        # It runs WITHOUT collectives -- another rank may be replaying a real step right now.
        state = (self.opt_g.flat_p, self.opt_g.flat_m, self.opt_g.flat_v, self.opt_g.hyper, self.opt_d.flat_p, self.opt_d.flat_m,
                 self.opt_d.flat_v, self.opt_d.hyper, ops.rng_state(sp.device))
        if self.vq_train:                        # the EMA moves the codebook buffers in every forward
            state += tuple(self.net_g.P(n) for n in CODEBOOK)
        snap = [t.clone() for t in state]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self.step(feed, collectives=False, **inj)
        torch.cuda.current_stream().wait_stream(side)
        for dst, src in zip(state, snap):
            dst.copy_(src)
        torch.cuda.synchronize()
        if self.vq_train:
            self.net_g.codebook_needs_init()     # the restore wrote `inited`: re-read it here, not during the capture
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        if self.world == 1:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=self._pool):
                r, loss_d = self._seg_a(feed, **inj)
                loss_g, parts = self._seg_b(r)
                self._seg_c()
            graphs = [graph]
        else:
            # world > 1: three graphs sharing the pool (replayed in capture order), collectives in between
            ga, gb, gc = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(ga, pool=self._pool):
                r, loss_d = self._seg_a(feed, **inj)
            with torch.cuda.graph(gb, pool=self._pool):
                loss_g, parts = self._seg_b(r)
            with torch.cuda.graph(gc, pool=self._pool):
                self._seg_c()
            graphs = [ga, gb, gc]
        out = self._outputs(loss_d, loss_g, parts, self.opt_d, self.opt_g)
        if keep:
            out["forward"] = {k: v for k, v in r.items() if torch.is_tensor(v)}
        return graphs, static, out

    def set_lr(self, lr):
        self.lr = lr
        self.opt_g.set_lr(lr)
        self.opt_d.set_lr(lr)

    def decay_lr(self):
        self.set_lr(self.lr * self.t["lr_decay"])


def synthetic_batch(B, T, X, device, seed=1234, hop=640, bank=None, ragged=False):
    """BASELINE config-3 shaped synthetic batch, generated on the HOST (pinned) like a DataLoader would deliver it,
    in the reference's collate layout (data_utils.py:167-226): ssl [B,768,T], wav [B,1,L], text [B,X]."""
    g = torch.Generator().manual_seed(seed)
    L = T * hop
    wav = (torch.rand(B, 1, L, generator=g) - 0.5)
    ssl = torch.randn(B, 768, T, generator=g)
    text = torch.randint(0, 732, (B, X), generator=g)
    if ragged:
        lengths = torch.randint(max(T // 2, 34), T + 1, (B,), generator=g)
        lengths[0] = T
        lengths, _ = torch.sort(lengths, descending=True)
        text_lengths = torch.randint(max(X // 2, 1), X + 1, (B,), generator=g)
        text_lengths[0] = X
    else:
        lengths = torch.full((B,), T, dtype=torch.long)
        text_lengths = torch.full((B,), X, dtype=torch.long)
    return dict(ssl=ssl, wav=wav, text=text, lengths=lengths, text_lengths=text_lengths)


def to_device_batch(host, device, bank, hop=640, vq_frames=None):
    """H2D + layout change + feature extraction that the reference does on CPU workers (data_utils.py:119-128):
    wav -> |X| on the GPU with the fused mel kernel.  Returns the channels-last dict S2Step consumes.
    vq_frames (the trainable quantizer only): the frame count of the reference collate's batch before any further padding;
    the batch then carries vq_rows = vq_frames // 2 as a device scalar."""
    wav = host["wav"].to(device, non_blocking=True)
    ssl = host["ssl"].to(device, non_blocking=True)
    text = host["text"].to(device, non_blocking=True)
    lengths = host["lengths"].to(device, non_blocking=True).to(torch.int32)
    text_lengths = host["text_lengths"].to(device, non_blocking=True).to(torch.int32)
    B, _, L = wav.shape
    # per-row sample counts (when the collate provides them): reflection at each utterance's own end (data_utils.py:119-128)
    lens = host["wav_lengths"].to(device, non_blocking=True).to(torch.int32) if "wav_lengths" in host else None
    spec, _ = ops.mel_frontend(wav.reshape(B, L), bank, hop, want_spec=True, want_mel=False, lens=lens)   # [B,T,1025], pitch 1028
    out = dict(ssl=ops.to_channels_last(ssl), spec=spec, lengths=lengths, wav=wav.reshape(B, L, 1), text=text,
               text_lengths=text_lengths)
    if vq_frames is not None:
        out["vq_rows"] = torch.tensor([vq_frames // 2], dtype=torch.int32).to(device, non_blocking=True)
    return out
