"""CPU tests of the host side of the stage-1 step on padded shapes: the DPO span draw plus a restatement of the device row
builder reproduce the reference's make_reject_y row for row (and leave the RNG where it left it), padding a collated batch
to the grid, and the two-rank gloo agreement on the padded shape."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

PAD = 1024


def _reference_make_reject_y(y_o, y_lens, generator=None):
    """utils.py:195-232 as the reference runs it (the repeat branch), with the draws inline."""
    rows, lens = [], []
    for b in range(len(y_lens)):
        y = y_o[b]
        i0, i1 = sorted(torch.randint(0, len(y), size=(2,), generator=generator).tolist())
        rows.append(torch.cat([y[:i0], y[i0:i1], y[i0:i1], y[i1:]]))
        lens.append(len(rows[-1]))
    out = torch.zeros((len(rows), max(lens)), dtype=y_o.dtype)
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out, torch.tensor(lens)


def _builder(y, spans, Yc, width):
    """evk_dpo_reject_rows restated: out[b][t] = y[b][t] (t < i1), y[b][t - (i1 - i0)] (t < Yc + i1 - i0), else 0."""
    B = y.shape[0]
    out = torch.zeros((B, width), dtype=torch.int64)
    lens = torch.zeros(B, dtype=torch.int64)
    for b in range(B):
        i0, i1 = int(spans[b, 0]), int(spans[b, 1])
        d, L = i1 - i0, Yc + i1 - i0
        for t in range(width):
            out[b, t] = y[b, t] if t < i1 else (y[b, t - d] if t < L else 0)
        lens[b] = L
    return out, lens


def _batch(B, Y, seed):
    g = torch.Generator().manual_seed(seed)
    yl = torch.randint(1, Y + 1, (B,), generator=g)
    yl[0] = Y
    y = torch.full((B, Y), PAD, dtype=torch.int64)
    for b in range(B):
        y[b, :yl[b]] = torch.randint(0, 1024, (int(yl[b]),), generator=g)
    return y, yl


@pytest.mark.parametrize("B,Y,seed", [(7, 23, 1), (12, 2, 2), (4, 150, 3), (1, 1, 4)])
def test_spans_and_builder_reproduce_make_reject_y(B, Y, seed):
    from easevoice_trainer_b200.models_gpt import make_reject_y, reject_spans, reject_width
    y, yl = _batch(B, Y, seed)
    g_ref, g_new, g_lib = (torch.Generator().manual_seed(seed + 100) for _ in range(3))
    ry, ryl = _reference_make_reject_y(y, yl, g_ref)
    spans = reject_spans(yl, Y, g_new)
    assert spans.dtype == torch.int32 and tuple(spans.shape) == (B, 2)
    W = reject_width(spans, Y)
    out, lens = _builder(torch.nn.functional.pad(y, (0, 9), value=PAD), spans, Y, W + 5)   # wider rows, padded width
    assert torch.equal(out[:, :W], ry) and (out[:, W:] == 0).all() and torch.equal(lens, ryl)
    r2, r2l = make_reject_y(y, yl, g_lib)
    assert torch.equal(r2, ry) and torch.equal(r2l, ryl)
    assert torch.equal(g_ref.get_state(), g_new.get_state()) and torch.equal(g_ref.get_state(), g_lib.get_state())


def test_default_generator_draws_are_unchanged():
    from easevoice_trainer_b200.models_gpt import make_reject_y
    y, yl = _batch(6, 40, 5)
    torch.manual_seed(17)
    ry, ryl = _reference_make_reject_y(y, yl)
    after = torch.get_rng_state()
    torch.manual_seed(17)
    r2, r2l = make_reject_y(y, yl)
    assert torch.equal(r2, ry) and torch.equal(r2l, ryl) and torch.equal(torch.get_rng_state(), after)


def test_builder_edge_spans():
    """i0 == i1 (nothing repeated), i1 == Yc (the tail repeated), the whole row, and an empty prefix."""
    y, _ = _batch(1, 12, 6)
    Yc = 12
    for i0, i1 in ((5, 5), (0, 0), (4, Yc), (0, Yc), (0, 3), (Yc, Yc)):
        ref = torch.cat([y[0, :i0], y[0, i0:i1], y[0, i0:i1], y[0, i1:]])
        out, lens = _builder(y, torch.tensor([[i0, i1]], dtype=torch.int32), Yc, 32)
        assert int(lens[0]) == len(ref) and torch.equal(out[0, :len(ref)], ref) and (out[0, len(ref):] == 0).all()


def test_pad_host_batch_to_grid():
    from easevoice_trainer_b200.train.data_gpt import pad_host_batch
    from easevoice_trainer_b200.train.gpt_step import quantize_len
    assert [quantize_len(n) for n in (0, 1, 32, 33, 64, 65)] == [0, 32, 32, 64, 64, 96]
    y, yl = _batch(3, 40, 7)
    x = torch.randint(0, 732, (3, 17))
    xl = torch.tensor([17, 9, 4])
    bert = torch.randn(3, 1024, 17)
    h = dict(ids=[0, 1, 2], phoneme_ids=x, phoneme_ids_len=xl, semantic_ids=y, semantic_ids_len=yl, bert_feature=bert)
    p = pad_host_batch(h, 32, 64)
    assert p["phoneme_ids"].shape == (3, 32) and p["semantic_ids"].shape == (3, 64) and p["bert_feature"].shape == (3, 1024, 32)
    assert torch.equal(p["phoneme_ids"][:, :17], x) and (p["phoneme_ids"][:, 17:] == 0).all()
    assert torch.equal(p["semantic_ids"][:, :40], y) and (p["semantic_ids"][:, 40:] == PAD).all()
    assert torch.equal(p["bert_feature"][..., :17], bert) and (p["bert_feature"][..., 17:] == 0).all()
    assert p["phoneme_ids_len"] is xl and p["semantic_ids_len"] is yl and p["ids"] == [0, 1, 2]
    assert pad_host_batch(h, 17, 40) is h


def _agree_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from easevoice_trainer_b200.train.gpt_step import GptStep

    class _S:                                   # only the shape agreement is exercised on CPU
        world = 2
        _shape_group = None
    s = _S()
    local = [(40, 100, 0), (70, 90, 150)][rank]
    ret[rank] = [GptStep.agree_shape(s, *local), GptStep.agree_shape(s, 33, 1, 0 if rank else 65)]
    dist.destroy_process_group()


def test_two_rank_gloo_shape_agreement_is_the_max():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_agree_worker, nprocs=2, args=(2, 29533, ret), join=True)
    assert ret[0] == ret[1] == [(96, 128, 160), (64, 32, 96)]
