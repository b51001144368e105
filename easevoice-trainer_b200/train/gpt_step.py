"""One stage-1 (AR semantic-token GPT) optimisation step on the sm_90a kernels.

Mirrors /root/reference/src/easevoice/soundstorm/auto_reg/models/t2s_lightning_module.py:
  training_step :41-89     manual optimisation: backward every micro-batch (loss is NOT divided), optimizer + scheduler
                           step when batch_idx > 0 and batch_idx % 4 == 0 (so the first update sees 5 micro-batches)
  configure_optimizers :91-124   ScaledAdam(lr=0.01, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=1000)
  lr_schedulers.py:36-65   the schedule is computed and then overridden: every scheduler.step() sets lr = end_lr (0.002);
                           the first optimizer step therefore runs at the constructor lr 0.01, all later ones at 0.002.
Differences that do not change the update: fp32 storage / TF32 tensor-core math instead of 16-mixed autocast; ScaledAdam
works on one flat arena (no per-step torch.stack / copy-back of every parameter, no `.item()` host syncs: optim.py:95-121,
:381); gradients accumulate in the flat buffer.  Data-parallel: NCCL all-reduce (mean, as DDP does) of the flat gradient
arena before the update.
"""
import torch
import torch.distributed as dist

from .. import ops
from ..models_gpt import reject_spans, reject_width

SCALED_ADAM_DEFAULTS = dict(lr=0.01, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=1000, scalar_lr_scale=0.1,
                            eps=1e-8, param_min_rms=1e-5, param_max_rms=3.0, scalar_max=10.0, size_update_period=4)
CHUNK = 8192
GRID = 32                # padded lengths (phonemes, semantic tokens, rejected rows) are rounded up to this many tokens


def quantize_len(n, q=GRID):
    return (int(n) + q - 1) // q * q


class FlatScaledAdam:
    """ScaledAdam state over flat fp32 arenas; the update is three launches of libevk (ops.scaled_adam)."""

    def __init__(self, named_params, **kw):
        self.cfg = dict(SCALED_ADAM_DEFAULTS, **kw)
        named = list(named_params)
        self.names = [n for n, _ in named]
        self.params = [p for _, p in named]
        dev = self.params[0].device
        total = sum(p.numel() for p in self.params)
        nt = len(self.params)
        self.flat_p = torch.empty(total, device=dev, dtype=torch.float32)
        self.flat_g = torch.zeros(total, device=dev, dtype=torch.float32)
        self.flat_delta = torch.zeros(total, device=dev, dtype=torch.float32)
        self.flat_v = torch.zeros(total, device=dev, dtype=torch.float32)
        self.slots, chunks, off = {}, [], 0
        for t, (n, p) in enumerate(named):
            k = p.numel()
            self.flat_p[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat_p[off:off + k].view_as(p)
            self.slots[n] = (off, k)
            for c in range(0, k, CHUNK):
                chunks.append((t, off + c, min(CHUNK, k - c)))
            off += k
        self.grad_views = [self.flat_g[o:o + k].view_as(p) for (o, k), p in zip(self.slots.values(), self.params)]
        self.chunks = torch.tensor(chunks, dtype=torch.int64, device=dev)
        self.numel = torch.tensor([p.numel() for p in self.params], dtype=torch.int64, device=dev)
        sup, per = self.cfg["size_update_period"], self.cfg["clipping_update_period"]
        f = dict(device=dev, dtype=torch.float32)
        self.stats, self.coef = torch.zeros(nt, 3, **f), torch.zeros(nt, 2, **f)
        self.rms, self.sv, self.sg = torch.zeros(nt, **f), torch.zeros(nt, **f), torch.zeros(sup, nt, **f)
        self.norms, self.thr, self.glob = torch.zeros(per, **f), torch.zeros(2, **f), torch.zeros(4, **f)
        self.hyper = torch.full((1,), float(self.cfg["lr"]), **f)
        self.stepbuf = torch.zeros(1, device=dev, dtype=torch.int64)

    @property
    def step_count(self):
        return int(self.stepbuf.item())

    def set_lr(self, lr):
        self.hyper.fill_(float(lr))

    def accumulate(self, grads):
        """flat_g += grads (micro-batch accumulation; None = parameter unused in this graph)."""
        views = [v for v, g in zip(self.grad_views, grads) if g is not None]
        torch._foreach_add_(views, [g for g in grads if g is not None])

    def step(self, gscale=1.0, zero_grad=True):
        ops.scaled_adam(self, gscale, zero_grad)

    def state_dict(self):
        """keys follow optim.py state names so a reference-side loader can map them tensor by tensor."""
        state = {}
        sc = self.step_count
        for i, n in enumerate(self.names):
            off, k = self.slots[n]
            shp = self.params[i].shape
            st = dict(step=sc, delta=self.flat_delta[off:off + k].view(shp).clone(), exp_avg_sq=self.flat_v[off:off + k].view(shp).clone())
            if k > 1:
                st.update(param_rms=self.rms[i].clone(), scale_exp_avg_sq=self.sv[i].clone(), scale_grads=self.sg[:, i].clone())
            state[i] = st
        return dict(state=state, names=list(self.names), model_norms=self.norms.clone(), model_norm_threshold=self.thr.clone(),
                    param_groups=[dict(self.cfg, lr=float(self.hyper.item()), params=list(range(len(self.names))))])

    def load_state_dict(self, sd):
        for i, n in enumerate(self.names):
            st = sd["state"].get(i)
            if st is None:
                continue
            off, k = self.slots[n]
            self.flat_delta[off:off + k].copy_(st["delta"].reshape(-1))
            self.flat_v[off:off + k].copy_(st["exp_avg_sq"].reshape(-1))
            if k > 1 and "param_rms" in st:
                self.rms[i] = st["param_rms"]; self.sv[i] = st["scale_exp_avg_sq"]; self.sg[:, i] = st["scale_grads"]
            self.stepbuf.fill_(int(st["step"]))
        # the clipping history is optional: states written by other ScaledAdam implementations (the reference keeps
        # `model_norms` inside the per-batch state, optim.py:330-346) simply restart the median-of-1000 window
        if "model_norms" in sd:
            self.norms.copy_(sd["model_norms"])
        if "model_norm_threshold" in sd:
            self.thr.copy_(sd["model_norm_threshold"])
        groups = sd.get("param_groups") or [{}]
        if "lr" in groups[0]:
            self.set_lr(groups[0]["lr"])


class GptStep:
    """Text2SemanticLightningModule.training_step for one micro-batch, graph-replayable."""

    ACCUM = 4
    LR_FIRST, LR_LOCKED = 0.01, 0.002          # lr_schedulers.py:36-65 (see module docstring)
    MAX_GRAPHS = 12          # LRU bound on the shapes train_step keeps captured (all graphs share one memory pool)
    CAPTURE_AFTER = 2        # train_step captures a shape the 2nd time it is seen; before that the eager step runs

    def __init__(self, model, world_size=1, dpo=False, **optim_kw):
        self.model, self.world, self.dpo = model, world_size, dpo
        self.lr = self.LR_FIRST
        self.opt = FlatScaledAdam(model.named_parameters(), **optim_kw)
        self.batch_idx = 0
        self._graph = None
        self._static = None
        self.last = None
        self._graphs = {}            # train_step: shape key -> (graph, static inputs, outputs); insertion order = LRU order
        self._seen = {}              # shape key -> sightings
        self._pool = None            # one private memory pool shared by every train_step graph
        self._opt_graph = None       # the ScaledAdam update, captured once in that pool (it does not depend on the shape)
        self._shape_group = None     # gloo group of the host-side shape agreement (world > 1)
        self.stats = dict(captures=0, replays=0, eager=0)

    # ---- eager pieces --------------------------------------------------------------------------
    def forward_backward(self, batch):
        """loss/acc + gradient accumulation for one micro-batch (no optimizer step).  A batch padded past the collate's
        shape (train_step) carries count = int32 device [2] (the collate's Y, the rejected rows' max length) and, for DPO,
        spans (int32 device [B, 2], reject_spans) and reject_width (the padded width of the rejected rows)."""
        m = self.model
        count = batch.get("count")
        if self.dpo:                                   # t2s_lightning_module.py:44 (if_dpo): CE + reference-free DPO term
            reject = batch.get("reject")
            if "spans" in batch:
                reject = ops.dpo_reject_rows(batch["semantic_ids"], batch["spans"], count[0:1], batch["reject_width"])
            loss, acc = m.forward(batch["phoneme_ids"], batch["phoneme_ids_len"], batch["semantic_ids"], batch["semantic_ids_len"],
                                  batch["bert_feature"], reject=reject,
                                  bert_channels_last=batch.get("bert_channels_last", False), count=count)
            with ops.grad_pool():
                grads = torch.autograd.grad(loss, self.opt.params, allow_unused=True)
                self.opt.accumulate(grads)
            return loss.detach(), acc
        loss, acc = m.forward_old(batch["phoneme_ids"], batch["phoneme_ids_len"], batch["semantic_ids"],
                                  batch["semantic_ids_len"], batch["bert_feature"], targets=batch.get("targets"),
                                  bert_channels_last=batch.get("bert_channels_last", False),
                                  count=None if count is None else count[0:1])
        with ops.grad_pool():
            grads = torch.autograd.grad(loss, self.opt.params, allow_unused=True)
            self.opt.accumulate(grads)
        return loss.detach(), acc

    def optimizer_step(self):
        if self.world > 1:
            dist.all_reduce(self.opt.flat_g)
        self.opt.step(gscale=1.0 / self.world, zero_grad=True)

    def wants_step(self):
        return self.batch_idx > 0 and self.batch_idx % self.ACCUM == 0

    def step(self, batch):
        """one training_step: micro-batch fwd/bwd, and the ScaledAdam update on every 4th batch index."""
        if self.model.training:
            ops.advance_rng()
        out = self.forward_backward(batch)
        if self.wants_step():
            self.optimizer_step()
            self.opt.set_lr(self.LR_LOCKED)
            self.lr = self.LR_LOCKED
        self.batch_idx += 1
        self.last = out
        return out

    # ---- CUDA-graph replay of the micro-batch (static shapes) -----------------------------------
    def _capture(self, batch):
        self._static = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
        m = self.model
        y_in, tg = m.make_targets(self._static["semantic_ids"], self._static["semantic_ids_len"].to(torch.int64))
        self._static["targets"] = (y_in, tg)
        snap = (self.opt.flat_g.clone(), ops.rng_state().clone())
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self.forward_backward(self._static)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            if m.training:
                ops.advance_rng()
            self._gout = self.forward_backward(self._static)
        self._ograph = torch.cuda.CUDAGraph()
        # the update graph is captured on a scratch copy of nothing: it only reads/writes optimizer arenas, and replaying
        # it during capture does not execute, so state is untouched here
        with torch.cuda.graph(self._ograph):
            self.opt.step(gscale=1.0 / self.world, zero_grad=True)
        self.opt.flat_g.copy_(snap[0])
        ops.rng_state().copy_(snap[1])

    def graph_step(self, batch):
        assert not self.dpo, "the DPO variant draws its rejected sequences on the host: use step()"
        if self._graph is None:
            self._capture(batch)
        for k, v in batch.items():
            if torch.is_tensor(v):
                self._static[k].copy_(v, non_blocking=True)
        y_in, tg = self.model.make_targets(self._static["semantic_ids"], self._static["semantic_ids_len"].to(torch.int64))
        self._static["targets"][0].copy_(y_in); self._static["targets"][1].copy_(tg)
        self._graph.replay()
        if self.wants_step():
            if self.world > 1:
                dist.all_reduce(self.opt.flat_g)
            self._ograph.replay()
            self.opt.set_lr(self.LR_LOCKED)
            self.lr = self.LR_LOCKED
        self.batch_idx += 1
        self.last = self._gout
        return self._gout

    # ---- padded shapes: grid, rank agreement and one graph per shape ------------------------------------------
    def agree_shape(self, X, Y, Yr=0):
        """-> (Xq, Yq, Yrq): the padded shape EVERY rank uses for this micro-batch.  Each rank's collate pads to its own
        batch maximum, so the local lengths (phonemes, semantic tokens, rejected rows; Yr = 0 without DPO) are rounded up
        to the GRID and MAX-reduced over a gloo (host-side) group: no GPU synchronisation, and all ranks capture, replay
        or fall back to the eager step at the same micro-batches, so their gradient all-reduces pair up."""
        q = [quantize_len(X), quantize_len(Y), quantize_len(Yr)]
        if self.world > 1:
            if self._shape_group is None:
                self._shape_group = dist.new_group(backend="gloo")
            t = torch.tensor(q, dtype=torch.int64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self._shape_group)
            q = [int(v) for v in t]
        return tuple(q)

    def prepare(self, host, device):
        """A collated host batch (data_gpt layout, pinned) -> the device batch train_step takes.  DPO spans are drawn
        here (reject_spans: the same torch.randint calls, in the same order, as make_reject_y in the eager forward); the
        batch is padded to the agreed shape and the counts + spans cross to the device in one pinned int32 buffer."""
        from .data_gpt import pad_host_batch
        Yc = host["semantic_ids"].shape[1]
        spans = reject_spans(host["semantic_ids_len"], Yc) if self.dpo else None
        Yr = reject_width(spans, Yc) if self.dpo else 0
        Xq, Yq, Yrq = self.agree_shape(host["phoneme_ids"].shape[1], Yc, Yr)
        host = pad_host_batch(host, Xq, Yq)
        meta = torch.tensor([Yc, Yr], dtype=torch.int32)
        if spans is not None:
            meta = torch.cat([meta, spans.reshape(-1)])
        meta = meta.pin_memory().to(device, non_blocking=True)
        batch = {k: host[k].to(device, non_blocking=True)
                 for k in ("phoneme_ids", "phoneme_ids_len", "semantic_ids", "semantic_ids_len", "bert_feature")}
        batch["count"] = meta[:2]
        if spans is not None:
            batch["spans"], batch["reject_width"] = meta[2:].view(-1, 2), Yrq
        return batch

    def train_step(self, batch):
        """What the trainer calls, on a batch from prepare(): replay the CUDA graph of this padded shape, capturing it
        the CAPTURE_AFTER-th time the shape shows up (at most MAX_GRAPHS kept, least recently used evicted); before that
        the eager step runs.  Same schedule, RNG stream and results as step() on the same batch."""
        key = (tuple(batch["phoneme_ids"].shape), tuple(batch["semantic_ids"].shape), batch.get("reject_width", 0))
        n = self._seen[key] = self._seen.get(key, 0) + 1
        if key not in self._graphs and n < self.CAPTURE_AFTER:
            self.stats["eager"] += 1
            return self.step(batch)
        g = self._graphs.pop(key, None)
        if g is None:
            while len(self._graphs) >= self.MAX_GRAPHS:
                self._graphs.pop(next(iter(self._graphs)))
            g = self._capture_shape(batch)
            self.stats["captures"] += 1
        else:
            self.stats["replays"] += 1
        self._graphs[key] = g                                            # (re)insert as most recently used
        graph, static, out = g
        for k, v in static.items():
            v.copy_(batch[k], non_blocking=True)
        graph.replay()
        if self.wants_step():
            if self.world > 1:
                dist.all_reduce(self.opt.flat_g)
            self._opt_graph.replay()
            self.opt.set_lr(self.LR_LOCKED)
            self.lr = self.LR_LOCKED
        self.batch_idx += 1
        self.last = out
        return out

    def _capture_shape(self, batch):
        static = {k: v.clone() for k, v in batch.items() if torch.is_tensor(v)}
        feed = dict(batch, **static)
        # warm-up (allocator, lazy initialisation) on a side stream; it must not count as training
        snap = (self.opt.flat_g.clone(), ops.rng_state().clone())
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self.forward_backward(feed)
        torch.cuda.current_stream().wait_stream(side)
        self.opt.flat_g.copy_(snap[0])
        ops.rng_state().copy_(snap[1])
        torch.cuda.synchronize()
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=self._pool):
            if self.model.training:
                ops.advance_rng()
            out = self.forward_backward(feed)
        if self._opt_graph is None:                  # captured, not run: the optimizer state is untouched
            self._opt_graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._opt_graph, pool=self._pool):
                self.opt.step(gscale=1.0 / self.world, zero_grad=True)
        return graph, static, out


def synthetic_batch(B=16, X=256, Y=1024, seed=0, device="cpu", ragged=False):
    """BASELINE.json configs[1]: batch 16, 1024 semantic tokens (+256 phonemes, 1024-d BERT features); pinned host memory
    when device == 'cpu' so bench.py's e2e leg can time the H2D copies (dataset.py:226-271 collate layout)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 732, (B, X), generator=g)
    y = torch.randint(0, 1024, (B, Y), generator=g)
    bert = torch.randn(B, 1024, X, generator=g)
    xl, yl = torch.full((B,), X, dtype=torch.int64), torch.full((B,), Y, dtype=torch.int64)
    if ragged:
        xl = torch.randint(max(X // 2, 1), X + 1, (B,), generator=g); xl[0] = X
        yl = torch.randint(max(Y // 2, 1), Y + 1, (B,), generator=g); yl[0] = Y
        for b in range(B):
            y[b, yl[b]:] = 1024
            bert[b, :, xl[b]:] = 0
    out = dict(phoneme_ids=x, phoneme_ids_len=xl, semantic_ids=y, semantic_ids_len=yl, bert_feature=bert)
    if device == "cpu":
        return {k: v.pin_memory() if torch.cuda.is_available() else v for k, v in out.items()}
    return {k: v.to(device) for k, v in out.items()}
