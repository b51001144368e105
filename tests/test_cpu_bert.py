"""BERT text features (Normalize.text / TextPreprocessor.get_bert_feature): the oracle reproduces the golden that
oracle/pin_bert.py produced from transformers and the reference's two callers, the checkpoint key mapping, and the host-side
checks and index map.  Nothing here needs a GPU: every input check of bert.py runs before its first library call."""
import os

import pytest
import torch

from oracle import bert_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = dict(vocab_size=40, hidden_size=64, num_hidden_layers=3, num_attention_heads=1, intermediate_size=128,
            max_position_embeddings=512)


def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "bert.pt"), weights_only=False)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("case", ["l4", "large"])
def test_oracle_matches_golden(case):
    g = _golden()[case]
    P = bert_oracle.init_params(bert_oracle.param_spec(g["cfg"]), g["seed"])
    for ids, w2p, feat, text in zip(g["input_ids"], g["word2ph"], g["features"], g["texts"]):
        assert len(ids) == len(text) + 2 and len(w2p) == len(text)
        h = bert_oracle.forward(P, g["cfg"], torch.tensor([ids]))
        f = bert_oracle.phone_level(h[0], w2p)
        assert f.shape == feat.shape == (g["cfg"]["hidden_size"], sum(w2p))
        assert _rel(f, feat) <= 1e-5


def _tiny_sd(prefix=""):
    from easevoice_trainer_b200 import bert
    net = bert.BertModel(TINY)
    return net, {prefix + k: torch.randn(v.shape) for k, v in net.state_dict().items()}


def test_state_dict_matches_oracle_spec():
    from easevoice_trainer_b200 import bert
    cfg = dict(bert_oracle.BERT_LARGE, **TINY)
    net = bert.BertModel(TINY)
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == bert_oracle.param_spec(cfg)


def test_key_mapping_prefix_gamma_beta_and_dropped_keys():
    net, sd = _tiny_sd()
    ck = {}
    for k, v in sd.items():
        k = k.replace("LayerNorm.weight", "LayerNorm.gamma").replace("LayerNorm.bias", "LayerNorm.beta")
        ck["bert." + k] = v
    ck["bert.embeddings.position_ids"] = torch.arange(512)[None]
    ck["bert.pooler.dense.weight"] = torch.randn(64, 64)
    ck["bert.pooler.dense.bias"] = torch.randn(64)
    ck["cls.predictions.bias"] = torch.randn(40)
    ck["cls.predictions.transform.LayerNorm.gamma"] = torch.randn(64)
    net.load_state_dict(ck)
    got = net.state_dict()
    assert set(got) == set(sd)
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    net2, sd2 = _tiny_sd()
    net2.load_state_dict(dict(sd2, **{"pooler.dense.weight": torch.randn(64, 64)}))      # unprefixed checkpoint
    assert torch.equal(net2.state_dict()["encoder.layer.2.output.dense.bias"], sd2["encoder.layer.2.output.dense.bias"])


def test_key_mapping_is_strict_otherwise():
    net, sd = _tiny_sd("bert.")
    with pytest.raises(RuntimeError):
        net.load_state_dict(dict(sd, **{"bert.encoder.layer.0.extra.weight": torch.zeros(1)}))
    sd.pop("bert.encoder.layer.1.intermediate.dense.bias")
    with pytest.raises(RuntimeError):
        net.load_state_dict(sd)


def test_config_rejects_other_activations_and_positions():
    from easevoice_trainer_b200 import bert
    with pytest.raises(ValueError):
        bert.BertModel(dict(TINY, hidden_act="gelu_new"))
    with pytest.raises(ValueError):
        bert.BertModel(dict(TINY, position_embedding_type="relative_key"))


class _CharTokenizer:
    """one token per character ([CLS] = 1, [SEP] = 2, characters 3..); `drop` characters are swallowed like an unknown
    whitespace, so fewer tokens come back than there are characters"""

    def __init__(self, drop=""):
        self.drop = drop

    def __call__(self, text, return_tensors="pt"):
        ids = [1] + [3 + (ord(c) % 30) for c in text if c not in self.drop] + [2]
        return {"input_ids": torch.tensor([ids]), "token_type_ids": torch.zeros(1, len(ids), dtype=torch.long),
                "attention_mask": torch.ones(1, len(ids), dtype=torch.long)}


def _cpu_model():
    from easevoice_trainer_b200 import bert
    return bert.BertModel(TINY)          # on the CPU: any library call would fail, so each error below comes from the checks


def test_word2ph_length_mismatch_raises():
    from easevoice_trainer_b200 import bert
    with pytest.raises(ValueError, match="word2ph"):
        bert.get_bert_feature("你好啊", [2, 2], _CharTokenizer(), _cpu_model())
    with pytest.raises(ValueError, match="word2ph"):
        bert.get_bert_features(["好", "你好啊"], [[2], [2, 2]], _CharTokenizer(), _cpu_model())


def test_character_past_the_tokens_raises():
    from easevoice_trainer_b200 import bert
    with pytest.raises(ValueError, match="no token"):
        bert.get_bert_feature("你 好", [2, 1, 2], _CharTokenizer(drop=" "), _cpu_model())


def test_more_than_512_tokens_raises():
    from easevoice_trainer_b200 import bert
    text = "字" * 511
    with pytest.raises(ValueError, match="max_position_embeddings"):
        bert.get_bert_feature(text, [1] * len(text), _CharTokenizer(), _cpu_model())
    with pytest.raises(ValueError, match="max_position_embeddings"):
        bert.get_bert_features(["好", text], [[1], [1] * len(text)], _CharTokenizer(), _cpu_model())
    with pytest.raises(ValueError, match="max_position_embeddings"):
        _cpu_model().hidden_state(torch.ones(1, 513, dtype=torch.long))


def test_attention_mask_must_be_a_prefix_of_ones():
    m = _cpu_model()
    ids = torch.ones(2, 5, dtype=torch.long)
    for mask in ([[1, 1, 0, 1, 0], [1, 1, 1, 1, 1]], [[0, 1, 1, 1, 1], [1, 1, 1, 1, 1]], [[1, 1, 1, 0, 0], [0, 0, 0, 0, 0]],
                 [[1, 1, 1, 1, 1]]):
        with pytest.raises(ValueError):
            m.hidden_state(ids, torch.tensor(mask))
    with pytest.raises(ValueError):
        m.hidden_state(ids, index=4)


def test_write_bert_features_checks_before_running(tmp_path):
    from easevoice_trainer_b200 import bert
    items = [("a.wav", "你好", [2, 2], 4, "zh"), ("b.wav", "你好", [2, 2], 5, "zh")]
    with pytest.raises(ValueError, match="b.wav.*phones"):
        bert.write_bert_features(items, str(tmp_path), _CharTokenizer(), _cpu_model())
    with pytest.raises(ValueError, match="c.wav.*word2ph"):
        bert.write_bert_features([("c.wav", "你好", [2], 2, "zh")], str(tmp_path), _CharTokenizer(), _cpu_model())
    # not zh, or already written: skipped, nothing to run
    (tmp_path / "d.wav.pt").write_bytes(b"x")
    assert bert.write_bert_features([("x.wav", "hi", [1], 9, "en"), ("d.wav", "你", [5], 0, "zh")], str(tmp_path),
                                    _CharTokenizer(), _cpu_model()) == []
    assert sorted(os.listdir(tmp_path)) == ["d.wav.pt"]


def test_phone_index_matches_repeat_interleave():
    from easevoice_trainer_b200 import bert
    w2ps = [[2, 1, 2, 0, 3], [1], [2, 2, 2, 1, 2, 2, 1]]
    T = 10
    idx, P = bert.phone_index(w2ps, T)
    assert P == [sum(w) for w in w2ps] and idx.shape == (3, max(P)) and idx.dtype == torch.long
    hidden = torch.randn(3, T, 16)
    flat = hidden.reshape(-1, 16)
    for b, w in enumerate(w2ps):
        want = torch.repeat_interleave(hidden[b, 1:1 + len(w)], torch.tensor(w), dim=0)
        assert torch.equal(flat[idx[b, :P[b]]], want)
        assert torch.equal(flat[idx[b, :P[b]]].T, bert_oracle.phone_level(hidden[b], w))
        assert bool((idx[b, P[b]:] == b * T).all())
