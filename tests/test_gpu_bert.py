"""GPU tests of the BERT text features (`pytest -m gpu`): the fused padded attention kernel (evk_attn_pad_fwd) against float64,
BertModel.hidden_state + phone_features against the features the reference computed (tests/golden/bert.pt, pinned by
oracle/pin_bert.py), batching and padding independence, and the Normalize.text writer."""
import json
import os

import pytest
import torch

from oracle import bert_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "bert.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
TOL_NET = 3e-3


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


class _precise:
    """3xTF32 products (evk_set_precise): comparisons between launches of different shapes, whose TF32 GEMMs may take
    different kernels, then show indexing errors instead of operand rounding"""

    def __enter__(self):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(1)

    def __exit__(self, *exc):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(0)


def _model(case):
    from easevoice_trainer_b200 import bert
    g = GOLD[case]
    net = bert.BertModel(g["cfg"])
    net.load_state_dict(bert_oracle.init_params(bert_oracle.param_spec(g["cfg"]), g["seed"]))
    return net.to(DEV).eval()


@pytest.fixture(scope="module")
def l4(ops):
    return _model("l4")


class _GoldTokenizer:
    """the tokenizer of oracle/pin_bert.py, replayed from the ids the golden keeps"""

    def __init__(self, case):
        self.ids = dict(zip(GOLD[case]["texts"], GOLD[case]["input_ids"]))

    def __call__(self, text, return_tensors="pt"):
        ids = self.ids[text]
        return {"input_ids": torch.tensor([ids]), "token_type_ids": torch.zeros(1, len(ids), dtype=torch.long),
                "attention_mask": torch.ones(1, len(ids), dtype=torch.long)}


@pytest.mark.parametrize("L", [1, 7, 63, 64, 65, 130, 512])
def test_attention_pad_kernel_against_float64(ops, L):
    from easevoice_trainer_b200 import lib
    B, H, D = 3, 16, 1024
    lens = [1, L, max(1, (2 * L) // 3)]
    g = torch.Generator().manual_seed(100 + L)
    qkv = torch.randn(B, L, 3 * D, generator=g).to(DEV)
    lens_d = torch.tensor(lens, device=DEV)
    c = qkv.double().cpu()
    want = []
    for b in range(B):
        q, k, v = [c[b, :, i * D:(i + 1) * D].view(L, H, 64).transpose(0, 1) for i in range(3)]
        s = (q @ k[:, :lens[b]].transpose(-1, -2)) / 8.0
        want.append((s.softmax(-1) @ v[:, :lens[b]]).transpose(0, 1).reshape(L, D))
    for precise, tol in ((0, 1e-3), (1, 2e-5)):
        lib.init().evk_set_precise(precise)
        try:
            out = ops.attention_pad(qkv, heads=H, lens=lens_d, scale=0.125)
            again = ops.attention_pad(qkv, heads=H, lens=lens_d, scale=0.125)
        finally:
            lib.init().evk_set_precise(0)
        torch.cuda.synchronize()
        assert torch.equal(out, again)                                   # no atomics: bit-reproducible
        assert bool(torch.isfinite(out).all())                           # rows at or past lens[b] included
        for b in range(B):
            assert rel(out[b, :lens[b]], want[b][:lens[b]]) <= tol, (precise, b)


def _features(net, case):
    from easevoice_trainer_b200 import bert
    g = GOLD[case]
    return [bert.get_bert_feature(t, w, _GoldTokenizer(case), net) for t, w in zip(g["texts"], g["word2ph"])]


@pytest.mark.parametrize("case", ["l4", "large"])
def test_features_match_golden(ops, case):
    net = _model(case)
    errs = []
    for f, want in zip(_features(net, case), GOLD[case]["features"]):
        assert f.device.type == "cuda" and f.dtype == torch.float32 and tuple(f.shape) == tuple(want.shape)
        errs.append(rel(f, want))
    print(f"bert golden {case}: rel-L2 per sentence {['%.2e' % e for e in errs]}")
    assert max(errs) <= TOL_NET, errs


def _padded(case):
    g = GOLD[case]
    n = [len(i) for i in g["input_ids"]]
    ids = torch.zeros((len(n), max(n)), dtype=torch.long)
    mask = torch.zeros_like(ids)
    for r, i in enumerate(g["input_ids"]):
        ids[r, :len(i)] = torch.tensor(i)
        mask[r, :len(i)] = 1
    return ids, mask, n


def test_batch_matches_each_sentence_alone_and_ignores_padding(l4):
    ids, mask, n = _padded("l4")
    with _precise():
        h = l4.hidden_state(ids, mask)
        errs = [rel(h[r, :n[r]], l4.hidden_state(torch.tensor([i]))[0]) for r, i in enumerate(GOLD["l4"]["input_ids"])]
    print(f"bert batch vs alone (3xTF32): rel-L2 {['%.2e' % e for e in errs]}")
    assert max(errs) <= 1e-5, errs
    h = l4.hidden_state(ids, mask)                                       # padding independence on the TF32 path
    g = torch.Generator().manual_seed(3)
    ids2 = torch.where(mask.bool(), ids, torch.randint(0, 21128, ids.shape, generator=g))
    h2 = l4.hidden_state(ids2, mask)
    for r in range(len(n)):
        assert torch.equal(h[r, :n[r]], h2[r, :n[r]]), r


def test_phone_features_are_exact_copies(l4):
    from easevoice_trainer_b200 import bert
    ids, mask, n = _padded("l4")
    w2ps = GOLD["l4"]["word2ph"]
    h = l4.hidden_state(ids, mask)
    f, P = bert.phone_features(h, w2ps)
    assert P == [sum(w) for w in w2ps] and tuple(f.shape) == (len(n), 1024, max(P))
    hc, fc = h.cpu(), f.cpu()
    for r, w in enumerate(w2ps):
        want = torch.repeat_interleave(hc[r, 1:1 + len(w)], torch.tensor(w), dim=0).T
        assert torch.equal(fc[r, :, :P[r]], want)
        assert not bool(fc[r, :, P[r]:].any())


def test_write_bert_features(l4, tmp_path):
    from easevoice_trainer_b200 import bert
    g = GOLD["l4"]
    tok = _GoldTokenizer("l4")
    t, w = g["texts"], g["word2ph"]
    keep = tmp_path / "b.pt"
    keep.write_bytes(b"already there")
    items = [("/data/a", t[0], w[0], sum(w[0]), "zh"), ("b", t[1], w[1], sum(w[1]), "zh"), ("c", t[2], w[2], sum(w[2]), "zh"),
             ("d", t[1], w[1], sum(w[1]), "en")]
    with _precise():
        assert bert.write_bert_features(items, str(tmp_path), tok, l4) == ["a", "c"]
        alone = {k: bert.get_bert_feature(t[k], w[k], tok, l4) for k in (0, 2)}
    assert sorted(os.listdir(tmp_path)) == ["a.pt", "b.pt", "c.pt"] and keep.read_bytes() == b"already there"
    for name, k in (("a", 0), ("c", 2)):
        f = torch.load(str(tmp_path / f"{name}.pt"), weights_only=False)
        assert f.device.type == "cpu" and f.dtype == torch.float32 and f.is_contiguous() and tuple(f.shape) == (1024, sum(w[k]))
        assert rel(f, alone[k]) <= 1e-5
        assert rel(f, g["features"][k]) <= TOL_NET
    with pytest.raises(ValueError, match="e.*phones"):
        bert.write_bert_features([("e", t[0], w[0], sum(w[0]) + 1, "zh")], str(tmp_path), tok, l4)


def test_from_pretrained_with_old_names_and_extra_keys(ops, tmp_path):
    from easevoice_trainer_b200 import bert
    g = GOLD["l4"]
    P = bert_oracle.init_params(bert_oracle.param_spec(g["cfg"]), g["seed"])
    sd = {}
    for k, v in P.items():
        sd["bert." + k.replace("LayerNorm.weight", "LayerNorm.gamma").replace("LayerNorm.bias", "LayerNorm.beta")] = v
    sd["bert.embeddings.position_ids"] = torch.arange(512)[None]
    sd["bert.pooler.dense.weight"] = torch.zeros(1024, 1024)
    sd["bert.pooler.dense.bias"] = torch.zeros(1024)
    sd["cls.predictions.bias"] = torch.zeros(21128)
    sd["cls.predictions.transform.dense.weight"] = torch.zeros(1024, 1024)
    torch.save(sd, str(tmp_path / "pytorch_model.bin"))
    (tmp_path / "config.json").write_text(json.dumps(dict(g["cfg"], architectures=["BertForMaskedLM"], hidden_act="gelu",
                                                          position_embedding_type="absolute", model_type="bert")))
    net = bert.BertModel.from_pretrained(str(tmp_path), device=DEV)
    assert net.cfg["num_hidden_layers"] == 4
    for f, want in zip(_features(net, "l4"), g["features"]):
        assert rel(f, want) <= TOL_NET
    (tmp_path / "config.json").write_text(json.dumps(dict(g["cfg"], hidden_act="relu")))
    with pytest.raises(ValueError):
        bert.BertModel.from_pretrained(str(tmp_path), device=DEV)
