#!/usr/bin/env python
"""Pin the BERT oracle (oracle/bert_oracle.py) against `transformers.BertForMaskedLM` and the reference's two unmodified callers
of it on the CPU, and write tests/golden/bert.pt.

  1. param_spec equals the `bert.*` part of BertForMaskedLM(config).state_dict(), names and shapes;
  2. with the seeded weights loaded into transformers, the oracle's forward matches hidden_states[-3] (max-abs <= 5e-5);
  3. the reference's Normalize._get_bert_feature (normalize.py:88-106) and TextPreprocessor.get_bert_feature
     (inference/preprocessor.py:180-193) return identical features, and the oracle's phone-level expansion matches them.

The tokenizer is a BertTokenizer over a small vocab written to a temporary directory; every hanzi of the test sentences must
tokenize to one token that is not [UNK].  The golden keeps the ids, so no test needs a tokenizer or transformers.  Cases:
  l4     4 layers (2 run) at full width, three sentences of 4, 13 and 37 characters
  large  the full 24-layer BERT-large config, one sentence of 20 characters

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_bert.py
"""
import importlib.util
import os
import random
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bert_oracle  # noqa: E402
from oracle.pin_against_reference import GOLD, REF, maxdiff  # noqa: E402
from oracle.ref_import import _stub  # noqa: E402

HANZI = "你好世界我们今天天气很不错中文语音合成的模型训练数据集准备文本特征提取声音说话人大家欢迎来到这里"
PUNCT = "，。！"
CASES = {
    "l4": dict(cfg=dict(bert_oracle.BERT_LARGE, num_hidden_layers=4), seed=5, text_seed=11, lengths=[4, 13, 37]),
    "large": dict(cfg=dict(bert_oracle.BERT_LARGE), seed=7, text_seed=12, lengths=[20]),
}


def make_tokenizer(tmp):
    from transformers import BertTokenizer
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + sorted(set(HANZI)) + list(PUNCT)
    path = os.path.join(tmp, "vocab.txt")
    with open(path, "w", encoding="utf8") as f:
        f.write("\n".join(vocab) + "\n")
    tok = BertTokenizer(vocab=path)          # transformers 5.x: the `vocab_file=` keyword is silently ignored
    for ch in set(HANZI) | set(PUNCT):
        ids = tok(ch, add_special_tokens=False)["input_ids"]
        assert len(ids) == 1 and ids[0] != tok.unk_token_id, (ch, ids)
    return tok


def make_texts(seed, lengths):
    """Sentences of hanzi with a punctuation mark every few characters and at the end; word2ph: 2 per hanzi, 1 per mark."""
    rnd = random.Random(seed)
    texts, w2ps = [], []
    for n in lengths:
        chars = [PUNCT[rnd.randrange(3)] if (i == n - 1 or (i > 0 and rnd.random() < 0.15)) else HANZI[rnd.randrange(len(HANZI))]
                 for i in range(n)]
        texts.append("".join(chars))
        w2ps.append([1 if c in PUNCT else 2 for c in chars])
    return texts, w2ps


def import_callers():
    """-> (Normalize, TextPreprocessor) from the unmodified reference modules; the imports their BERT methods do not use are
    replaced by empty stand-ins."""
    sys.path.insert(0, REF)
    for n in ("librosa", "LangSegment"):
        _stub(n)
    _stub("src.utils.config", torch=torch)           # normalize.py takes `torch` from this module's star import
    _stub("src.utils.audio", load_audio=None)
    _stub("src.utils.helper", random_choice=None, get_hparams_from_file=None)
    _stub("src.easevoice.feature_extractor.cnhubert", CNHubert=None)
    _stub("src.easevoice.module.models", SynthesizerTrn=None)
    _stub("src.easevoice.text.cleaner", clean_text=None)
    _stub("src.easevoice.text", cleaned_text_to_sequence=None, chinese=None)
    _stub("src.easevoice.inference").__path__ = [os.path.join(REF, "src", "easevoice", "inference")]
    _stub("src.easevoice.inference.segmentation", SPLITS=set(), PUNCTUATION=set(), split_big_text=None, get_split_method=None)
    mods = []
    for name, rel in (("src.normalization.normalize", "src/normalization/normalize.py"),
                      ("src.easevoice.inference.preprocessor", "src/easevoice/inference/preprocessor.py")):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
        m = importlib.util.module_from_spec(spec)
        sys.modules[name] = m
        spec.loader.exec_module(m)
        mods.append(m)
    return mods[0].Normalize, mods[1].TextPreprocessor


def transformers_model(cfg, P):
    from transformers import BertConfig, BertForMaskedLM
    conf = BertConfig(**cfg, hidden_act="gelu", position_embedding_type="absolute", hidden_dropout_prob=0.0,
                      attention_probs_dropout_prob=0.0)
    model = BertForMaskedLM(conf).eval()
    sd = model.state_dict()
    bert = {k[len("bert."):]: tuple(v.shape) for k, v in sd.items() if k.startswith("bert.") and not k.endswith(".position_ids")}
    assert bert == {k: tuple(s) for k, s in bert_oracle.param_spec(cfg).items()}, sorted(set(bert) ^ set(bert_oracle.param_spec(cfg)))
    missing, unexpected = model.load_state_dict({"bert." + k: v for k, v in P.items()}, strict=False)
    assert not unexpected and all(k.startswith("cls.") for k in missing), (missing, unexpected)
    return model


def pin_case(name, case, tok, Normalize, TextPreprocessor):
    cfg = case["cfg"]
    P = bert_oracle.init_params(bert_oracle.param_spec(cfg), case["seed"])
    model = transformers_model(cfg, P)
    pre = TextPreprocessor(model, tok, torch.device("cpu"))
    texts, w2ps = make_texts(case["text_seed"], case["lengths"])
    ids, feats, err_h, err_f = [], [], 0.0, 0.0
    for text, w2p in zip(texts, w2ps):
        enc = tok(text, return_tensors="pt")
        assert enc["input_ids"].shape[1] == len(text) + 2 and int(enc["token_type_ids"].abs().sum()) == 0
        with torch.no_grad():
            hs = model(**enc, output_hidden_states=True)["hidden_states"]
        ho = bert_oracle.forward(P, cfg, enc["input_ids"], enc["attention_mask"])
        err_h = max(err_h, maxdiff(ho, hs[-3]))
        resp = Normalize._get_bert_feature(None, text, w2p, tok, model)
        f_norm = resp.data["phone_level_feature"]
        f_pre = pre.get_bert_feature(text, w2p)
        assert torch.equal(f_norm, f_pre), maxdiff(f_norm, f_pre)
        assert f_norm.shape == (cfg["hidden_size"], sum(w2p))
        err_f = max(err_f, maxdiff(bert_oracle.phone_level(ho[0], w2p), f_norm))
        ids.append(enc["input_ids"][0].tolist())
        feats.append(f_norm.contiguous().clone())
    assert err_h <= 5e-5 and err_f <= 5e-5, (err_h, err_f)
    return dict(cfg=cfg, seed=case["seed"], texts=texts, input_ids=ids, word2ph=w2ps, features=feats), dict(
        max_abs_oracle_vs_transformers=err_h, max_abs_phone_features=err_f, phones=[sum(w) for w in w2ps])


if __name__ == "__main__":
    import transformers
    torch.manual_seed(0)
    Normalize, TextPreprocessor = import_callers()
    gold, report = {"transformers": transformers.__version__}, {}
    with tempfile.TemporaryDirectory() as tmp:
        tok = make_tokenizer(tmp)
        for name, case in CASES.items():
            gold[name], report[name] = pin_case(name, case, tok, Normalize, TextPreprocessor)
    torch.save(gold, os.path.join(GOLD, "bert.pt"))
    print(report)
