"""GPU tests of the stage-1 step on padded shapes (`pytest -m gpu`): the device builder of the DPO rejected rows, the counted-length
bound of the CE / DPO losses (the loss at the 32-token grid equals the loss at the collate's shape), GptStep.train_step's CUDA
graphs against the eager step (bit for bit, plain and DPO, across optimizer updates and LRU eviction), and GPTTrain end to end
on train_step with checkpoints that load like the reference's."""
import contextlib
import io
import math
import os
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
PAD = 1024


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


def _model(layer_dropout, n_layer=2, seed=7):
    from easevoice_trainer_b200.configs import GPT_MODEL
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    return Text2SemanticDecoder({"model": dict(GPT_MODEL, n_layer=n_layer)}, layer_dropout=layer_dropout, seed=seed).to(DEV).train()


def _host_batch(B, X, Y, seed):
    """A collated host batch (Text2SemanticDataset.collate layout, pinned) with ragged lengths; row 0 has the full X / Y."""
    g = torch.Generator().manual_seed(seed)
    xl = torch.randint(max(X // 2, 1), X + 1, (B,), generator=g); xl[0] = X
    yl = torch.randint(max(Y // 2, 1), Y + 1, (B,), generator=g); yl[0] = Y
    x = torch.zeros((B, X), dtype=torch.int64)
    y = torch.full((B, Y), PAD, dtype=torch.int64)
    bert = torch.zeros((B, 1024, X))
    for b in range(B):
        x[b, :xl[b]] = torch.randint(0, 732, (int(xl[b]),), generator=g)
        y[b, :yl[b]] = torch.randint(0, 1024, (int(yl[b]),), generator=g)
        bert[b, :, :xl[b]] = torch.randn(1024, int(xl[b]), generator=g)
    out = dict(phoneme_ids=x, phoneme_ids_len=xl, semantic_ids=y, semantic_ids_len=yl, bert_feature=bert)
    return {k: v.pin_memory() for k, v in out.items()}


def _flat_grad(loss, net):
    return torch.cat([g.reshape(-1) for g in torch.autograd.grad(loss, list(net.parameters()))])


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def test_reject_builder_matches_make_reject_y(ops):
    from easevoice_trainer_b200.models_gpt import make_reject_y, reject_spans, reject_width
    from easevoice_trainer_b200.train.gpt_step import quantize_len
    for B, Y, seed in ((5, 37, 1), (12, 3, 2), (3, 200, 3)):                  # Y = 3: spans with i0 == i1 are common
        h = _host_batch(B, 8, Y, seed)
        y, yl = h["semantic_ids"], h["semantic_ids_len"]
        ry, ryl = make_reject_y(y, yl, torch.Generator().manual_seed(seed))       # host path: the reference's rows
        spans = reject_spans(yl, Y, torch.Generator().manual_seed(seed))
        W = reject_width(spans, Y)
        assert W == ry.shape[1]
        Wq = quantize_len(W)
        yc = torch.tensor([Y], dtype=torch.int32, device=DEV)
        out, lens = ops.dpo_reject_rows(torch.nn.functional.pad(y, (0, 32), value=PAD).to(DEV), spans.to(DEV), yc, Wq)
        torch.testing.assert_close(out.cpu(), torch.nn.functional.pad(ry, (0, Wq - W)), rtol=0, atol=0)
        torch.testing.assert_close(lens.cpu(), ryl, rtol=0, atol=0)
        ryd, ryld = make_reject_y(y.to(DEV), yl.to(DEV), torch.Generator().manual_seed(seed))   # device path of make_reject_y
        torch.testing.assert_close(ryd.cpu(), ry, rtol=0, atol=0)
        torch.testing.assert_close(ryld.cpu(), ryl, rtol=0, atol=0)


def _padded(h, Xq, Yq):
    from easevoice_trainer_b200.train.data_gpt import pad_host_batch
    return {k: v.to(DEV) for k, v in pad_host_batch(h, Xq, Yq).items()}


@pytest.mark.parametrize("dpo", [False, True])
def test_counted_loss_at_grid_shape_equals_collate_shape(ops, dpo):
    """Dropout off: the loss at the padded grid shape with counts is the loss at the collate's shape (1e-5 relative), and so
    is the flat gradient (1e-4 rel-L2).  Under 3xTF32 products: with one TF32 product per MAC, padding the text changes the
    GEMM tiling and so which sums' operands round differently, which alone moves the flat gradient by up to ~5e-4 rel-L2."""
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1)
    try:
        _counted_loss_case(ops, dpo)
    finally:
        lib.init().evk_set_precise(0)


def _counted_loss_case(ops, dpo):
    from easevoice_trainer_b200.models_gpt import reject_spans, reject_width
    from easevoice_trainer_b200.train.gpt_step import quantize_len
    net = _model(0.0)
    B, X, Y = 6, 41, 90
    h = _host_batch(B, X, Y, 11)
    Xq, Yq = quantize_len(X) + 32, quantize_len(Y) + 32                        # one grid cell further than needed as well
    d0 = {k: v.to(DEV) for k, v in h.items()}
    dq = _padded(h, Xq, Yq)
    count = torch.tensor([Y, 0], dtype=torch.int32, device=DEV)
    if not dpo:
        l0, a0 = net.forward_old(d0["phoneme_ids"], d0["phoneme_ids_len"], d0["semantic_ids"], d0["semantic_ids_len"], d0["bert_feature"])
        g0 = _flat_grad(l0, net)
        lq, aq = net.forward_old(dq["phoneme_ids"], dq["phoneme_ids_len"], dq["semantic_ids"], dq["semantic_ids_len"], dq["bert_feature"],
                                 count=count[0:1])
        gq = _flat_grad(lq, net)
    else:
        spans = reject_spans(h["semantic_ids_len"], Y, torch.Generator().manual_seed(5))
        W = reject_width(spans, Y)
        count[1] = W
        yc = count[0:1]
        r0 = ops.dpo_reject_rows(d0["semantic_ids"], spans.to(DEV), yc, W)
        l0, a0 = net.forward(d0["phoneme_ids"], d0["phoneme_ids_len"], d0["semantic_ids"], d0["semantic_ids_len"], d0["bert_feature"],
                             reject=r0)
        g0 = _flat_grad(l0, net)
        rq = ops.dpo_reject_rows(dq["semantic_ids"], spans.to(DEV), yc, quantize_len(W) + 32)
        lq, aq = net.forward(dq["phoneme_ids"], dq["phoneme_ids_len"], dq["semantic_ids"], dq["semantic_ids_len"], dq["bert_feature"],
                             reject=rq, count=count)
        gq = _flat_grad(lq, net)
    el = abs(float(lq.detach()) - float(l0.detach())) / abs(float(l0.detach()))
    eg = _rel_l2(gq, g0)
    print(f"{'dpo' if dpo else 'forward_old'}: loss {float(l0.detach()):.6f} vs {float(lq.detach()):.6f} rel {el:.2e}; acc {float(a0):.6f} vs "
          f"{float(aq):.6f}; flat grad rel-L2 {eg:.2e}")
    assert el <= 1e-5
    assert eg <= 1e-4
    assert abs(float(aq) - float(a0)) <= 1e-6


def _state(step):
    o = step.opt
    return [o.flat_p, o.flat_delta, o.flat_v, o.flat_g, o.rms, o.sv, o.sg, o.norms, o.thr, o.stepbuf, o.hyper]


def _run_arm(dpo, hosts, graphs, max_graphs=None, capture_after=None):
    """Fresh model + GptStep, seeded RNGs; every host batch through prepare() and then train_step (graphs) or step()."""
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.train.gpt_step import GptStep
    net = _model(0.1)
    step = GptStep(net, dpo=dpo)
    if max_graphs is not None:
        step.MAX_GRAPHS = max_graphs
    if capture_after is not None:
        step.CAPTURE_AFTER = capture_after
    torch.manual_seed(123)                                   # the reject spans' draws
    ops.manual_seed(99)
    rec = []
    for h in hosts:
        b = step.prepare(h, DEV)
        loss, acc = step.train_step(b) if graphs else step.step(b)
        rec.append((loss.clone(), acc.clone()))
    torch.cuda.synchronize()
    return rec, [t.clone() for t in _state(step)], step


def _assert_same_run(a, b):
    (ra, sa, _), (rb, sb, _) = a, b
    for i, ((la, aa), (lb, ab)) in enumerate(zip(ra, rb)):
        assert torch.equal(la, lb) and torch.equal(aa, ab), (i, float(la), float(lb), float(aa), float(ab))
    names = ["flat_p", "flat_delta", "flat_v", "flat_g", "rms", "sv", "sg", "norms", "thr", "stepbuf", "hyper"]
    for n, x, y in zip(names, sa, sb):
        assert torch.equal(x, y), n


@pytest.mark.parametrize("dpo", [False, True])
def test_train_step_bit_identical_to_eager_step(ops, dpo):
    """Dropout on: 9 micro-batches of one grid cell (two optimizer updates) through train_step (eager, capture, replays) and
    through the eager step on the same padded batches: losses, accuracies, parameters and the ScaledAdam state are equal bit
    for bit.  DPO batches differ in their rejected width, so their graphs are captured on first sight."""
    hosts = [_host_batch(4, 40 + 3 * i, 100 + 3 * i, 100 + i) for i in range(9)]    # all in the cell (64, 128)
    eager = _run_arm(dpo, hosts, graphs=False)
    graph = _run_arm(dpo, hosts, graphs=True, capture_after=1 if dpo else None)
    st = graph[2].stats
    print(f"dpo={dpo}: {st}, optimizer steps {graph[2].opt.step_count}")
    assert graph[2].opt.step_count == 2 and st["captures"] >= 1 and st["captures"] + st["replays"] >= 8
    _assert_same_run(eager, graph)


def test_lru_eviction_and_recapture_bit_identical(ops):
    """Three grid cells with room for two graphs: evicted shapes are captured again and the run stays equal to the eager one."""
    cells = [(40, 70), (70, 110), (100, 200)]                   # grid cells (64, 96), (96, 128), (128, 224)
    order = [0, 0, 1, 1, 2, 2, 0, 1, 2, 0, 2, 1]
    hosts = [_host_batch(3, cells[c][0] - i % 3, cells[c][1] - i % 5, 300 + i) for i, c in enumerate(order)]
    eager = _run_arm(False, hosts, graphs=False)
    graph = _run_arm(False, hosts, graphs=True, max_graphs=2)
    st = graph[2].stats
    print(f"lru: {st}")
    assert len(graph[2]._graphs) == 2 and st["captures"] >= 5 and st["eager"] == 3
    _assert_same_run(eager, graph)


def test_gpttrain_epoch_on_train_step_and_checkpoints_load(ops):
    """GPTTrain on a tiny synthetic project runs one epoch through train_step; its trainer checkpoint and half-precision export
    have the layout the reference's loaders take (tests/golden/ckpt_layouts.json) and load back strictly."""
    import yaml
    from collections import OrderedDict
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    from easevoice_trainer_b200.train import data_gpt
    from easevoice_trainer_b200.train.gpt import GPTTrain, GPTTrainParams, GPT_CONFIG_PATH
    from easevoice_trainer_b200.train.gpt_step import FlatScaledAdam
    from tests.test_cpu_ckpt_roundtrip import _check_layout
    rnd = torch.Generator().manual_seed(11)
    with tempfile.TemporaryDirectory() as td:
        inp = os.path.join(td, "in"); os.makedirs(os.path.join(inp, "3-bert"))
        with open(os.path.join(inp, "2-name2text.txt"), "w") as f2, open(os.path.join(inp, "6-name2semantic.tsv"), "w") as f6:
            f6.write("item_name\tsemantic_audio\n")
            for i in range(12):
                nph = int(torch.randint(8, 40, (1,), generator=rnd))
                nsem = int(nph * 25 / float(torch.randint(5, 12, (1,), generator=rnd)))
                f2.write(f"utt{i}\t" + " ".join(f"p{int(v)}" for v in torch.randint(0, 732, (nph,), generator=rnd)) + "\tw2p\tnorm text\n")
                f6.write(f"utt{i}\t" + " ".join(str(int(v)) for v in torch.randint(0, 1024, (nsem,), generator=rnd)) + "\n")
                torch.save(torch.randn(1024, nph, generator=rnd), os.path.join(inp, "3-bert", f"utt{i}.pt"))
        ds = data_gpt.Text2SemanticDataset(os.path.join(inp, "2-name2text.txt"), os.path.join(inp, "6-name2semantic.tsv"),
                                           max_sec=54, phoneme_table={f"p{i}": i for i in range(732)})
        params = GPTTrainParams(batch_size=12, total_epochs=1, save_every_epoch=1, gpu_ids="0", model_path="", train_input_dir=inp,
                                output_model_name="tiny", project_dir=td)
        trainer = GPTTrain(params, dataset=ds, config_path=GPT_CONFIG_PATH)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            res = trainer.train()
        st = trainer.gpt_step.stats
        rec = [l for l in buf.getvalue().splitlines() if l.startswith("loss-of-easevoice")]
        print(f"GPTTrain: {len(rec)} steps, {st}")
        assert len(rec) == sum(st.values()) and st["captures"] + st["replays"] > 0
        ck = os.listdir(os.path.join(res.model_path, "logs", "ckpt"))
        assert len(ck) == 1 and ck[0].startswith("epoch=0-step=")
        sd = torch.load(os.path.join(res.model_path, "logs", "ckpt", ck[0]), map_location="cpu", weights_only=False)
        _check_layout(sd["state_dict"].items(), "t2s_state")
        w = torch.load(os.path.join(res.model_path, "tiny-e1.ckpt"), map_location="cpu", weights_only=False)
        _check_layout(w["weight"].items(), "t2s_state")
        assert all(v.dtype == torch.float16 for v in w["weight"].values()) and w["info"] == "GPT-e1"
        config = yaml.safe_load(open(GPT_CONFIG_PATH))
        net = Text2SemanticDecoder(config, top_k=3)
        net.load_state_dict(OrderedDict((k[len("model."):], v.float()) for k, v in w["weight"].items()), strict=True)
        net.load_state_dict(OrderedDict((k[len("model."):], v) for k, v in sd["state_dict"].items()), strict=True)
        opt = FlatScaledAdam(net.named_parameters())
        opt.load_state_dict(sd["optimizer_states"][0])
        assert opt.step_count == sd["global_step"] and all(math.isfinite(float(v)) for v in sd["state_dict"]["model.ar_predict_layer.weight"].reshape(-1)[:16])
