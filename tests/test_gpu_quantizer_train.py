"""Trainable semantic quantizer (freeze_quantizer: false) on the GPU: the vq_train.cu kernels against the reference-pinned
golden (tests/golden/s2_quantizer_train.pt) and the CPU oracle, and the stage-2 step with the quantizer unfrozen (graph
replay, resume, data parallel)."""
import os

import pytest
import torch

from oracle import vq_train_oracle as O
from tests import checks

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s2_quantizer_train.pt")
CB = "quantizer.vq.layers.0._codebook."
BUFS = ("embed", "embed_avg", "cluster_size", "inited")


@pytest.fixture(scope="module")
def evk():
    from easevoice_trainer_b200 import lib
    L = lib.init()
    L.evk_set_precise(0)
    return L


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


def _cl(t):
    return t.transpose(1, 2).contiguous().cuda()


@pytest.mark.parametrize("grid_pad", [0, 32], ids=["reference_shape", "padded_grid"])
def test_kernels_match_reference_golden(evk, grid_pad):
    """Three training forwards from a zero codebook: codes bit-exact, buffers within TOL_F32, kl_ssl within 1e-5, ssl_proj
    gradients under the NET_GRAD rule.  padded_grid appends 32 frames that must not touch any statistic."""
    from easevoice_trainer_b200 import ops
    gold = torch.load(GOLD, weights_only=False)
    c, run = gold["cfg"], gold["run"]
    w0, b0, ssls, ups = O.pin_inputs(c)
    w, b = w0.cuda().requires_grad_(True), b0.cuda().requires_grad_(True)
    buf = dict(embed=torch.zeros(c["K"], c["D"]), embed_avg=torch.zeros(c["K"], c["D"]), cluster_size=torch.zeros(c["K"]),
               inited=torch.zeros(1))
    buf = {k: v.cuda() for k, v in buf.items()}
    T2 = c["T"] // 2
    rows = torch.tensor([T2], dtype=torch.int32, device="cuda")
    for i, (ssl, up, ref) in enumerate(zip(ssls, ups, run["steps"])):
        ssl = torch.nn.functional.pad(ssl, (0, grid_pad))
        up = torch.nn.functional.pad(up, (0, grid_pad))
        x = ops.ssl_proj_fp32(_cl(ssl), w, b)
        if i == 0:
            ops.vq_kmeans_init_(x, rows, buf["embed"], buf["embed_avg"], buf["cluster_size"], buf["inited"], idx=run["kmeans_idx"])
        with torch.no_grad():
            codes = ops.vq_nearest(x, buf["embed"])
            q = ops.embedding(buf["embed"], codes)
            ops.vq_ema_(x, codes, rows, buf["cluster_size"], buf["embed_avg"], buf["embed"])
        y, kl = ops.vq_straight_through(x, q, rows)
        dw, db = torch.autograd.grad((y * _cl(up)).sum() + kl, [w, b])
        assert torch.equal(codes[:, :T2].cpu(), ref["codes"].reshape(c["B"], T2)), i
        assert abs(float(kl.detach()) - float(ref["kl_ssl"])) <= 1e-5 * abs(float(ref["kl_ssl"])), (i, float(kl.detach()), float(ref["kl_ssl"]))
        for k in ("embed", "embed_avg", "cluster_size"):
            assert _rel(buf[k], ref["buffers"][k]) <= checks.TOL_F32, (i, k, _rel(buf[k], ref["buffers"][k]))
        assert float(buf["inited"]) == 1.0
        ew, eb = _rel(dw, ref["dweight"]), _rel(db, ref["dbias"])
        assert ew <= checks.NET_GRAD_TENSOR and eb <= checks.NET_GRAD_TENSOR, (i, ew, eb)


def test_kmeans_integer_bit_exact(evk):
    """Integer samples (exact distances and means, many tied duplicates): means and bins equal the reference's bit for bit."""
    from easevoice_trainer_b200 import ops
    ik = torch.load(GOLD, weights_only=False)["kmeans_int"]
    x = ik["samples"].cuda().unsqueeze(0)                        # one batch row of 40 frames
    K, D = ik["means"].shape
    emb, ea, cs, ini = torch.zeros(K, D, device="cuda"), torch.zeros(K, D, device="cuda"), torch.zeros(K, device="cuda"), torch.zeros(1, device="cuda")
    rows = torch.tensor([x.shape[1]], dtype=torch.int32, device="cuda")
    ops.vq_kmeans_init_(x, rows, emb, ea, cs, ini, idx=ik["idx"])
    assert torch.equal(emb.cpu(), ik["means"]) and torch.equal(ea.cpu(), ik["means"])
    assert torch.equal(cs.cpu(), ik["bins"].float()) and float(ini) == 1.0


# ---- the stage-2 step with the quantizer unfrozen -------------------------------------------------------------------
def _setup(lr=None):
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.train import s2_step
    from oracle import s2_oracle
    net_g, net_d, _, _ = checks._load_models()
    net_g.freeze_quantizer = False
    with torch.no_grad():
        for n in BUFS:
            net_g.P(CB + n).zero_()
    net_g.train(); net_d.train()
    st = s2_step.S2Step(net_g, net_d, dict(s2_oracle.S2_TRAIN), dict(s2_oracle.S2_DATA))
    if lr is not None:
        st.set_lr(lr)
    ops.manual_seed(77)
    return st


def _batches(st, n, T=48):
    from easevoice_trainer_b200.train import s2_step
    out = []
    for i in range(n):
        host = s2_step.synthetic_batch(2, T, 12, "cuda", seed=100 + i)
        out.append(s2_step.to_device_batch(host, torch.device("cuda", 0), st.bank, vq_frames=T))
    return out


def _state(st):
    return {n: st.net_g.P(CB + n).clone() for n in BUFS}


def test_step_buffers_vs_oracle(evk):
    """lr 0: the step's codebook after 1 and 3 steps (the first from inited = 0) against the oracle; kl_ssl within 1e-5;
    ssl_proj now trains in the base group (it gets a gradient and enters grad_norm_g)."""
    st = _setup(lr=0.0)
    g = torch.Generator().manual_seed(5)
    idx = torch.randint(0, 48, (1024,), generator=g)
    batches = _batches(st, 3)
    w = st.net_g.P("ssl_proj.weight").detach().cpu().clone()
    b = st.net_g.P("ssl_proj.bias").detach().cpu().clone()
    buf = {k: v.cpu() for k, v in _state(st).items()}
    for i, batch in enumerate(batches):
        out = st.step(batch, kmeans_idx=idx if i == 0 else None)
        ssl = batch["ssl"].transpose(1, 2).cpu()
        r = O.step(ssl, w, b, buf, torch.zeros_like(ssl), kmeans_idx=idx)
        buf = r["buffers"]
        if i in (0, 2):
            for k in ("embed", "embed_avg", "cluster_size"):
                e = _rel(st.net_g.P(CB + k), buf[k])
                assert e <= checks.TOL_F32, (i, k, e)
            assert float(st.net_g.P(CB + "inited")) == 1.0
        assert abs(float(out["kl_ssl"]) - float(r["kl_ssl"])) <= 1e-5 * abs(float(r["kl_ssl"])), (i, float(out["kl_ssl"]))
    off, k = st.opt_g.slots["ssl_proj.weight"]
    assert off + k <= st.opt_g.n_active and float(st.opt_g.flat_g[off:off + k].abs().max()) > 0.0


def test_graph_step_equals_eager_step(evk):
    batches = _batches(_setup(), 3)
    eager = _setup()
    outs_e = [float(eager.step(b)["kl_ssl"]) for b in batches]
    graph = _setup()
    outs_g = [float(graph.step(batches[0])["kl_ssl"])] + [float(graph.graph_step(b)["kl_ssl"]) for b in batches[1:]]
    for k, v in _state(eager).items():
        assert _rel(_state(graph)[k], v) <= 1e-6, k
    assert _rel(graph.opt_g.flat_p, eager.opt_g.flat_p) <= 1e-6
    for oe, og in zip(outs_e, outs_g):
        assert abs(og - oe) <= 1e-6 * abs(oe), (outs_e, outs_g)


def test_resume_continues_the_ema(evk, tmp_path):
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.utils import ckpt
    batches = _batches(_setup(), 3)
    a = _setup()
    for bt in batches:
        a.step(bt)
    b = _setup()
    b.step(batches[0])
    rng = ops.rng_state().clone()
    path = str(tmp_path / "G_1.pth")
    ckpt.save_checkpoint(b.net_g, b.opt_g, 1e-4, 1, path)
    ckpt.save_checkpoint(b.net_d, b.opt_d, 1e-4, 1, str(tmp_path / "D_1.pth"))
    c = _setup()
    ckpt.load_checkpoint(path, c.net_g, c.opt_g)
    ckpt.load_checkpoint(str(tmp_path / "D_1.pth"), c.net_d, c.opt_d)
    assert not c.net_g.codebook_needs_init()
    ops.rng_state().copy_(rng)
    for bt in batches[1:]:
        c.step(bt)
    for k, v in _state(a).items():
        assert _rel(_state(c)[k], v) <= 1e-6, k
    assert _rel(c.opt_g.flat_p, a.opt_g.flat_p) <= 1e-6


def _two_rank_worker(rank, world, port, result):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from easevoice_trainer_b200 import lib
        from easevoice_trainer_b200.train import s2_step
        from oracle import s2_oracle
        lib.init()
        net_g, net_d, _, _ = checks._load_models()
        net_g.freeze_quantizer = False
        net_g.train(); net_d.train()
        st = s2_step.S2Step(net_g, net_d, dict(s2_oracle.S2_TRAIN), dict(s2_oracle.S2_DATA), world_size=world)
        host = s2_step.synthetic_batch(2, 48, 12, "cuda", seed=200 + rank)     # different data on every rank
        batch = s2_step.to_device_batch(host, torch.device("cuda", rank), st.bank, vq_frames=48)
        st.step(batch)
        st.step(batch)
        emb = net_g.P(CB + "embed").clone()
        mine = emb.clone()
        dist.broadcast(emb, src=0)
        st._broadcast_codebook()
        result[rank] = bool(torch.equal(net_g.P(CB + "embed"), emb)) and (rank == 0 or not torch.equal(mine, emb))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_share_rank0_codebook(evk):
    """DDP(broadcast_buffers=True) semantics: before every G forward rank 0's codebook replaces the others', so after a step
    each rank's own EMA differs, and the next broadcast gives every rank rank 0's codebook."""
    import random
    import torch.multiprocessing as mp
    result = mp.Manager().dict()
    mp.spawn(_two_rank_worker, nprocs=2, args=(2, random.randint(30000, 55000), result))
    assert result[0] and result[1], dict(result)
