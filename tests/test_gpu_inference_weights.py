"""GPU tests of the packed-weight cache of the inference models (`pytest -m gpu`): a second call in the same precise mode packs
nothing, and a model that ran with TF32 products and is then switched to 3xTF32 (evk_set_precise) computes the same bits as a
fresh model in that mode, for Whisper (whose decode step is a captured graph), BERT and the stage-1 GPT decoder."""
import json
import os

import pytest
import torch

from oracle import bert_oracle, gpt_oracle
from oracle import pin_asr as PIN

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)


@pytest.fixture
def packs(monkeypatch):
    """[number of ops.pack_weight calls so far]"""
    from easevoice_trainer_b200 import ops
    n, real = [0], ops.pack_weight

    def counted(*a, **k):
        n[0] += 1
        return real(*a, **k)
    monkeypatch.setattr(ops, "pack_weight", counted)
    return n


def _same(a, b):
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.cpu(), b.cpu())
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _switch_to_precise(make, run, packs):
    """run(net) twice with TF32 products, then twice under 3xTF32 on the same net: the second call of each mode packs
    nothing, and the 3xTF32 result is that of a fresh net in that mode (and not the TF32 result)."""
    from easevoice_trainer_b200 import lib
    L = lib.init()
    L.evk_set_precise(0)
    try:
        net = make()
        tf32 = run(net)
        n = packs[0]
        assert n > 0 and _same(run(net), tf32) and packs[0] == n
        L.evk_set_precise(1)
        got = run(net)
        n = packs[0]
        assert _same(run(net), got) and packs[0] == n
        want = run(make())
    finally:
        L.evk_set_precise(0)
    assert not _same(tf32, want)
    assert _same(got, want)


def test_whisper_switch_to_precise(packs):
    from easevoice_trainer_b200 import whisper
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "asr.pt"), weights_only=False)
    c = gold["cases"]["m80_d2"]
    xs = [PIN.clip(c["seed"] * 10 + i, s) for i, s in enumerate(c["secs"])]
    wav = torch.zeros(len(xs), max(x.size for x in xs))
    for i, x in enumerate(xs):
        wav[i, :x.size] = torch.from_numpy(x)
    wav = wav.to(DEV)

    def make():
        net = whisper.WhisperModel(c["cfg"], gold["gen"])
        net.load_state_dict(PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"]))
        return net.to(DEV).eval()

    def run(net):
        feats = net.features(wav, [x.size for x in xs])
        enc = net.encode(feats)
        return enc, net.transcribe_features(feats, language="en", enc=enc)
    _switch_to_precise(make, run, packs)


def test_bert_switch_to_precise(packs):
    from easevoice_trainer_b200 import bert
    g = torch.load(os.path.join(ROOT, "tests", "golden", "bert.pt"), weights_only=False)["l4"]
    ids = g["input_ids"]
    n = max(len(i) for i in ids)
    mask = torch.tensor([[1] * len(i) + [0] * (n - len(i)) for i in ids])
    ids = torch.tensor([i + [0] * (n - len(i)) for i in ids])

    def make():
        net = bert.BertModel(g["cfg"])
        net.load_state_dict(bert_oracle.init_params(bert_oracle.param_spec(g["cfg"]), g["seed"]))
        return net.to(DEV).eval()
    _switch_to_precise(make, lambda net: net.hidden_state(ids, mask), packs)


def test_gpt_switch_to_precise(packs):
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    c = json.load(open(os.path.join(ROOT, "tests", "golden", "infer_batch.json")))["cfg"]
    m = dict(gpt_oracle.GPT_MODEL, n_layer=4)
    gen = torch.Generator().manual_seed(c["seed"])
    x = [torch.randint(0, 732, (n,), generator=gen).to(DEV) for n in c["x_lens"]]
    bert_f = [torch.randn(1024, n, generator=gen).to(DEV) for n in c["x_lens"]]
    prompts = torch.randint(0, 1024, (1, c["Yp"]), generator=gen).expand(c["B"], -1).to(DEV)

    def make():
        net = Text2SemanticDecoder({"model": m})
        net.load_state_dict(gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), c["param_seed"]))
        return net.to(DEV).eval()

    def run(net):
        trace = []
        y, idx = net.infer_panel_batch_infer(x, torch.tensor(c["x_lens"]), prompts, bert_f, top_k=1, early_stop_num=20,
                                             trace=trace)
        return trace, y, idx
    _switch_to_precise(make, run, packs)
