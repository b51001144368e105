#!/usr/bin/env python
"""Throughput of the AR decoding loop (SURVEY 8 row f4, AR half): Text2SemanticDecoder.infer_panel at the reference's model size
(24 layers, d = 512), 120 phonemes + 150 prompt tokens, 300 generated tokens (early_stop_num), top_k 15 / top_p 1 / T 1 as TTS
calls it.  CPU arm: the reference-equivalent KV-cache loop restated with torch ops on this box's cores (bounded: 40 tokens).
One JSON line.   python tools/bench_infer_panel.py > gpurun_out/bench_infer_panel.json"""
# --batch: instead, the same single-utterance number next to infer_panel_batch_infer for B in {1, 4, 16} sentences (each with the
# same 120 phonemes / 150-token prompt / 300 tokens), as aggregate semantic tokens/s and ms per decoding step, with the card's
# name and power limit read in the same run.  --profile DIR (with --batch): also a torch.profiler trace of one B = 16 call.
# --ref-free: prompt-free decoding (TTS's ref_text_free mode), infer_panel_naive(prompts=None) on one utterance next to
# infer_panel_naive_batched(prompts=None) for B in {1, 4, 16}, same 120 phonemes / 300 tokens / top_k 15, card name and power limit.
# --new N: N generated tokens (early_stop_num) instead of 300 in every mode, e.g. 40 for a short sentence, where the steps run
# past a batch's last finish between two reads of the finished flags weigh the most.
# --precision float16|bfloat16 (with --batch or --ref-free): the batched numbers for the fp32 and the 16-bit compute type
# (Text2SemanticDecoder.set_compute_type), alternated twice in one process, each with its peak allocated memory; with --profile
# DIR, instead only the torch.profiler trace and per-kernel table of one B = 16 call in the 16-bit compute type.
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from easevoice_trainer_b200 import lib  # noqa: E402
from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder  # noqa: E402
from oracle import gpt_oracle  # noqa: E402  (CPU arm: parameter init + the cached loop below)

lib.init()
dev = torch.device("cuda", 0)
m = dict(gpt_oracle.GPT_MODEL)
P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), 35)
net = Text2SemanticDecoder({"model": m})
net.load_state_dict(P)
net = net.to(dev).eval()
X, Yp = 120, 150
NEW = int(sys.argv[sys.argv.index("--new") + 1]) if "--new" in sys.argv else 300
g = torch.Generator().manual_seed(2)
x = torch.randint(0, m["phoneme_vocab_size"], (1, X), generator=g)
bert = torch.randn(1, 1024, X, generator=g)
prompts = torch.randint(0, 1024, (1, Yp), generator=g)
xd, bd, pd, xl = x.to(dev), bert.to(dev), prompts.to(dev), torch.tensor([X], device=dev)
BATCH = "--batch" in sys.argv
REF_FREE = "--ref-free" in sys.argv
PREC = {"float16": torch.float16, "bfloat16": torch.bfloat16}[sys.argv[sys.argv.index("--precision") + 1]] if "--precision" in sys.argv else None


def card_name():
    import subprocess
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    return card[0] if card else "unknown"


def profile_b16(d):
    """torch.profiler trace and per-kernel table of one B = 16 infer_panel_batch_infer call (40 tokens), after a warm-up"""
    os.makedirs(d, exist_ok=True)
    B = 16
    args = ([xd[0]] * B, torch.full((B,), X), pd.expand(B, -1), [bd[0]] * B)
    net.infer_panel_batch_infer(*args, top_k=15, top_p=1, early_stop_num=40, temperature=1.0)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        net.infer_panel_batch_infer(*args, top_k=15, top_p=1, early_stop_num=40, temperature=1.0)
        torch.cuda.synchronize()
    tag = "" if net.compute_type is None else "_" + str(net.compute_type).split(".")[-1]
    prof.export_chrome_trace(os.path.join(d, f"infer_batch_b16{tag}.pt.trace.json"))
    with open(os.path.join(d, f"infer_batch_b16{tag}_kernels.txt"), "w") as f:
        f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))


def bench_ref_free():
    """infer_panel_naive(prompts=None) on one utterance and infer_panel_naive_batched(prompts=None) for B in {1, 4, 16}: generated
    tokens / wall time of one call (prompt pass included)."""
    net.infer_panel_naive(xd, xl, None, bd, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)            # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    y, _ = net.infer_panel_naive(xd, xl, None, bd, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    single = dict(tokens_per_s=y.shape[1] / s, ms_per_token=s / max(y.shape[1], 1) * 1e3, generated=int(y.shape[1]))
    out = {}
    for B in (1, 4, 16):
        xs, bs, lens = [xd[0]] * B, [bd[0]] * B, torch.full((B,), X)
        net.infer_panel_naive_batched(xs, lens, None, bs, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)  # warm-up, capture
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ys, _ = net.infer_panel_naive_batched(xs, lens, None, bs, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        gen = [int(t.shape[0]) for t in ys]
        steps = max(gen) + 1
        out[str(B)] = dict(tokens_per_s=sum(gen) / s, ms_per_step=s / steps * 1e3, generated=sum(gen), steps=steps, seconds=s)
    return single, out


if REF_FREE and PREC is None:
    single, batch = bench_ref_free()
    print(json.dumps(dict(metric="Text2SemanticDecoder.infer_panel_naive_batched(prompts=None) (prompt-free batched KV-cache AR decoding)",
                          unit="semantic-tokens/s", card=card_name(), single_utterance=single, batch=batch,
                          config=dict(layers=24, X=X, prompt=0, early_stop_num=NEW, top_k=15, top_p=1, temperature=1.0),
                          note="aggregate generated tokens over wall time of one call, prompt pass included; 25 tokens = 1 s of audio")))
    sys.exit(0)


def bench_batch():
    """infer_panel_batch_infer for B in {1, 4, 16}: aggregate generated tokens / wall time (prompt pass included)."""
    out = {}
    for B in (1, 4, 16):
        xs, bs, ps = [xd[0]] * B, [bd[0]] * B, pd.expand(B, -1)
        lens = torch.full((B,), X)
        net.infer_panel_batch_infer(xs, lens, ps, bs, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)      # warm-up, capture
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ys, idx = net.infer_panel_batch_infer(xs, lens, ps, bs, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        gen = [int(y.shape[0]) - Yp for y in ys]
        steps = max(gen) + 1
        out[str(B)] = dict(tokens_per_s=sum(gen) / s, ms_per_step=s / steps * 1e3, generated=sum(gen), steps=steps, seconds=s)
    if "--profile" in sys.argv and PREC is None:
        profile_b16(sys.argv[sys.argv.index("--profile") + 1])
    return out, card_name()


if PREC is not None and (BATCH or REF_FREE):
    if "--profile" in sys.argv:
        net.set_compute_type(PREC)
        profile_b16(sys.argv[sys.argv.index("--profile") + 1])
        sys.exit(0)
    card, arms = card_name(), []
    for dt in (None, PREC, None, PREC):
        net.set_compute_type(dt)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        if BATCH:
            arms.append(dict(compute_type=str(dt), batch=bench_batch()[0]))
        else:
            single, batch = bench_ref_free()
            arms.append(dict(compute_type=str(dt), single_utterance=single, batch=batch))
        arms[-1]["peak_allocated_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    print(json.dumps(dict(metric="Text2SemanticDecoder " + ("infer_panel_naive_batched(prompts=None)" if REF_FREE else "infer_panel_batch_infer")
                          + ": fp32 against the 16-bit compute type, alternated", unit="semantic-tokens/s", card=card, arms=arms,
                          config=dict(layers=24, X=X, prompt=0 if REF_FREE else Yp, early_stop_num=NEW, top_k=15, top_p=1, temperature=1.0),
                          note="aggregate generated tokens over wall time of one call, prompt pass included; 25 tokens = 1 s of audio")))
    sys.exit(0)


# every warm-up runs at the timed size: it packs the weights, sizes the KV caches and captures the step graph, so that the timed
# call measures decoding alone
net.infer_panel(xd, xl, pd, bd, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)
torch.cuda.synchronize()
t0 = time.perf_counter()
y, idx = net.infer_panel(xd, xl, pd, bd, top_k=15, top_p=1, early_stop_num=NEW, temperature=1.0)
torch.cuda.synchronize()
gpu_s = time.perf_counter() - t0
new = y.shape[1] - Yp


def cpu_cached_decode(n_new):
    """process_prompt + decode_next_token (t2s_model.py:121-221) with torch CPU ops, greedy, n_new tokens"""
    D, H, dk = 512, 16, 32
    pe = gpt_oracle.sine_pe(X + Yp + n_new + 2, D)
    xe = F.embedding(x, P["ar_text_embedding.word_embeddings.weight"]) + F.linear(bert.transpose(1, 2), P["bert_proj.weight"], P["bert_proj.bias"])
    xe = xe + P["ar_text_position.alpha"] * pe[:X]
    ye = F.embedding(prompts, P["ar_audio_embedding.word_embeddings.weight"]) + P["ar_audio_position.alpha"] * pe[:Yp]
    h = torch.cat([xe, ye], 1)
    mask = gpt_oracle.prefix_lm_mask(torch.tensor([X]), torch.tensor([Yp]), X, Yp)
    add = torch.zeros(mask.shape).masked_fill(mask, float("-inf")).unsqueeze(1)
    kc, vc = [], []

    def block(i, h, add_, kcache=None, vcache=None):
        p = f"h.layers.{i}."
        qkv = F.linear(h, P[p + "self_attn.in_proj_weight"], P[p + "self_attn.in_proj_bias"])
        q, k, v = qkv.split(D, dim=-1)
        if kcache is not None:
            k, v = torch.cat([kcache, k], 1), torch.cat([vcache, v], 1)
        L, Lk = q.shape[1], k.shape[1]
        qh, kh, vh = q.view(1, L, H, dk).transpose(1, 2), k.view(1, Lk, H, dk).transpose(1, 2), v.view(1, Lk, H, dk).transpose(1, 2)
        s = qh @ kh.transpose(-2, -1) / math.sqrt(dk)
        att = torch.softmax(s + add_ if add_ is not None else s, -1) @ vh
        att = F.linear(att.transpose(1, 2).reshape(1, L, D), P[p + "self_attn.out_proj.weight"], P[p + "self_attn.out_proj.bias"])
        h = F.layer_norm(h + att, (D,), P[p + "norm1.weight"], P[p + "norm1.bias"], 1e-5)
        ff = F.linear(torch.relu(F.linear(h, P[p + "linear1.weight"], P[p + "linear1.bias"])), P[p + "linear2.weight"], P[p + "linear2.bias"])
        return F.layer_norm(h + ff, (D,), P[p + "norm2.weight"], P[p + "norm2.bias"], 1e-5), k, v
    for i in range(m["n_layer"]):
        h, k, v = block(i, h, add)
        kc.append(k); vc.append(v)
    last = h[:, -1:]
    for t in range(n_new):
        tok = F.linear(last[:, 0], P["ar_predict_layer.weight"])[:, :-1].argmax(-1, keepdim=True)
        last = F.embedding(tok, P["ar_audio_embedding.word_embeddings.weight"]) + P["ar_audio_position.alpha"] * pe[Yp + t]
        for i in range(m["n_layer"]):
            last, kc[i], vc[i] = block(i, last, None, kc[i], vc[i])


if BATCH:
    batch, card = bench_batch()
    print(json.dumps(dict(metric="Text2SemanticDecoder.infer_panel_batch_infer (batched KV-cache AR decoding)", unit="semantic-tokens/s",
                          card=card, single_utterance=dict(tokens_per_s=new / gpu_s, ms_per_token=gpu_s / max(new, 1) * 1e3, generated=new),
                          batch=batch, config=dict(layers=24, X=X, prompt=Yp, early_stop_num=NEW, top_k=15, top_p=1, temperature=1.0),
                          note="aggregate generated tokens over wall time of one call, prompt pass included; 25 tokens = 1 s of audio")))
    sys.exit(0)
threads = min(16, os.cpu_count() or 1)
torch.set_num_threads(threads)
n_cpu = 40
with torch.no_grad():
    t0 = time.perf_counter()
    cpu_cached_decode(n_cpu)
    cpu_s = time.perf_counter() - t0
print(json.dumps(dict(metric="Text2SemanticDecoder.infer_panel (KV-cache AR decoding), one utterance", unit="semantic-tokens/s",
                      value=new / gpu_s, generated=new, seconds=gpu_s, ms_per_token=gpu_s / max(new, 1) * 1e3,
                      config=dict(layers=24, X=X, prompt=Yp, early_stop_num=NEW, top_k=15, top_p=1, temperature=1.0),
                      note="prompt pass included in the time; 25 tokens = 1 s of audio",
                      cpu_baseline=dict(value=n_cpu / cpu_s, unit="semantic-tokens/s", cores=threads, kind="port",
                                        sample=f"prompt pass + {n_cpu} greedy tokens, torch CPU ops, KV cache as t2s_model.py:121-221"))))
