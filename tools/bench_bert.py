#!/usr/bin/env python
"""Speed of the BERT text features (SURVEY 8 row f3, text half; the TTS text front end) with seeded BERT-large weights
(24 layers, 1024 wide; hidden_states[-3], so 22 layers run).  One JSON line:

  tts_segment       one 30-character sentence, B = 1: ms per get_bert_feature call, host ids to device features
  normalize_text    512 seeded sentences of 8-60 characters through get_bert_features, D2H of every feature included
  attention         evk_attn_pad_fwd against ops.attention (batched GEMMs + softmax) at (B, L) = (1, 32) and (32, 64), 16 heads
  cpu_baseline      the oracle forward of the TTS sentence on the host's CPU cores (the reference runs this step on the CPU)
  transformers_gpu  BertForMaskedLM in fp32 on the same GPU (as the reference TTS runs it), when transformers is importable

The card's name and power limit are read in the same run.  The tokenizer is a per-character stand-in (one id per character),
so tokenization is not part of any figure.
   python tools/bench_bert.py > bench_bert.json"""
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from easevoice_trainer_b200 import bert, lib, ops  # noqa: E402
from oracle import bert_oracle as bo  # noqa: E402  (CPU arm + seeded weights)

HANZI = "你好世界我们今天天气很不错中文语音合成的模型训练数据集准备文本特征提取声音说话人大家欢迎来到这里"


class CharTokenizer:
    def __call__(self, text, return_tensors="pt"):
        ids = [101] + [672 + (ord(c) * 7919) % 20000 for c in text] + [102]
        return {"input_ids": torch.tensor([ids]), "token_type_ids": torch.zeros(1, len(ids), dtype=torch.long)}


def sentence(rnd, n):
    return "".join("，" if (i % 9 == 8 or i == n - 1) else rnd.choice(HANZI) for i in range(n))


def w2p(text):
    return [1 if c == "，" else 2 for c in text]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def event_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    lib.init().evk_set_precise(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    cfg = dict(bo.BERT_LARGE)
    P = bo.init_params(bo.param_spec(cfg), 42)
    net = bert.BertModel(cfg)
    net.load_state_dict(P)
    net = net.to(dev).eval()
    tok = CharTokenizer()
    rnd = random.Random(5)

    # TTS segment: one 30-character sentence
    seg = sentence(rnd, 30)
    seg_ids = tok(seg)["input_ids"]
    for _ in range(5):
        f = bert.get_bert_feature(seg, w2p(seg), tok, net)
    seg_s = timed(lambda: bert.get_bert_feature(seg, w2p(seg), tok, net), 50)

    # Normalize.text: 512 sentences of 8..60 characters
    texts = [sentence(rnd, rnd.randint(8, 60)) for _ in range(512)]
    w2ps = [w2p(t) for t in texts]
    n_tok = sum(len(t) + 2 for t in texts)

    def corpus():
        return [x.cpu() for x in bert.get_bert_features(texts, w2ps, tok, net)]
    corpus()
    norm_s = min(timed(corpus, 1) for _ in range(3))

    # attention alone
    attn = {}
    with torch.no_grad():
        for B, L in ((1, 32), (32, 64)):
            g = torch.Generator().manual_seed(B * 1000 + L)
            qkv = torch.randn(B, L, 3 * 1024, generator=g).to(dev)
            lens = torch.full((B,), L, dtype=torch.long, device=dev)
            klen = lens.int()
            fused = lambda: ops.attention_pad(qkv, heads=16, lens=lens, scale=0.125)      # noqa: E731
            mat = lambda: ops.attention(qkv[..., :1024], qkv[..., 1024:2048], qkv[..., 2048:], heads=16, scale=0.125,  # noqa: E731
                                        klen=klen)
            for _ in range(20):
                fused(); mat()
            ms_f, ms_m = [], []
            for _ in range(3):                                   # alternate the two arms
                ms_f.append(event_ms(fused, 200))
                ms_m.append(event_ms(mat, 200))
            err = float((fused() - mat()).norm() / mat().norm())
            attn[f"B{B}_L{L}"] = dict(fused_us=min(ms_f) * 1e3, materialised_us=min(ms_m) * 1e3,
                                      speedup=min(ms_m) / min(ms_f), rel_l2_fused_vs_materialised=err)

    # CPU arm: the oracle forward of the TTS sentence
    threads = min(16, os.cpu_count() or 1)
    torch.set_num_threads(threads)
    t0 = time.perf_counter()
    hc = bo.forward(P, cfg, seg_ids)
    cpu_s = time.perf_counter() - t0
    fc = bo.phone_level(hc[0], w2p(seg))
    f = bert.get_bert_feature(seg, w2p(seg), tok, net).cpu()
    err_cpu = float((f.double() - fc.double()).norm() / fc.double().norm())

    # transformers on the same GPU, fp32
    hf = None
    try:
        from transformers import BertConfig, BertForMaskedLM
        conf = BertConfig(**cfg, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
        m = BertForMaskedLM(conf).eval()
        m.load_state_dict({"bert." + k: v for k, v in P.items()}, strict=False)
        m = m.to(dev)

        def hf_call():
            with torch.no_grad():
                res = m(input_ids=seg_ids.to(dev), output_hidden_states=True)["hidden_states"][-3][0][1:-1]
            return torch.cat([res[i].repeat(w, 1) for i, w in enumerate(w2p(seg))], 0).T
        for _ in range(5):
            hf_call()
        hf_s = timed(hf_call, 50)
        hf = dict(ms=hf_s * 1e3, rel_l2_vs_library=float((hf_call().cpu().double() - f.double()).norm() / f.double().norm()))
        del m
    except ImportError:
        pass

    print(json.dumps(dict(
        metric="BERT-large text features (hidden_states[-3], 22 of 24 layers), seeded weights", gpu=name, power_limit=power,
        tts_segment=dict(chars=30, tokens=32, phones=sum(w2p(seg)), ms=seg_s * 1e3),
        normalize_text=dict(sentences=len(texts), tokens=n_tok, s=norm_s, utt_per_s=len(texts) / norm_s, tokens_per_s=n_tok / norm_s),
        attention=attn,
        cpu_baseline=dict(ms=cpu_s * 1e3, cores=threads, kind="oracle forward, one 30-character sentence"),
        transformers_gpu=hf, rel_l2_vs_cpu_oracle=err_cpu)))


if __name__ == "__main__":
    main()
