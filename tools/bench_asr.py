#!/usr/bin/env python
"""Whisper transcription throughput on one GPU (whisper.py), against transformers' `generate(num_beams=5)` on the same GPU.

Workload: seeded large-v3-shaped weights (d_model 1280, 32 + 32 layers, 128 mel bins, 51 866 tokens; 1.55 G parameters) and
`--clips` seeded clips of 2-12 s at 32 kHz (tones under noise), resampled to 16 kHz on the device as `WhisperAsr` does.
Random weights seldom emit eot, so the generation config here suppresses eot and every clip decodes a fixed budget of
ceil(--tokens-per-second x its length) tokens (8-48 at the default 4 tokens/s).  Clips are sorted by length and batched
(equal batches within `asr.clips_per_batch`'s 16 GiB default); a batch decodes the largest budget of its clips, in both arms.

Reports one JSON line: audio-seconds/s end to end (front end + encoder + decode, device-synchronised host clock), peak
device memory, the device-time split (front end, encoder, cross K/V, decode steps; the beam step's share of a step from one
profiled eager step), the encoder's TFLOP/s from shapes, and the comparator arms (fp32 with TF32 allowed and fp16, one clip per
call and batched) on the first `--compare-clips` clips.  The card's name and power limit are read in the same run.

--long: long-form transcription (`WhisperModel.transcribe_long`) of `--clips` (default 8) seeded 16 kHz clips of 40-300 s in
one pool, every 30 s window decoding `--tokens-per-window` tokens (eot suppressed, as above); reports audio-seconds/s end
to end, the device-time split (whole-clip front end, encoder, decode), peak memory and the comparator: transformers'
long-form `generate` (attention_mask, temperature 0, logprob / no-speech thresholds) on the same features, fp32 with TF32 and
fp16, batched.

--precision float16|bfloat16: the short-form measurement twice for each of the fp32 (TF32) and the 16-bit compute type on
one model, alternating fp32, 16-bit, fp32, 16-bit in the same process.  Each arm adds the Linears' device time in one profiled
eager decode step, their share of the step and the floor of that time: the step's Linear weight bytes (shapes below) over
3.35 TB/s of HBM3.

Usage:  python tools/bench_asr.py [--clips 256] [--compare-clips 16] [--no-compare] [--precision float16|bfloat16]
        python tools/bench_asr.py --long [--clips 8] [--tokens-per-window 120] [--no-compare]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def generation_config():
    """large-v3's special-token layout: eot 50257, sot 50258, 100 languages, <|notimestamps|> 50364, 1501 timestamps."""
    langs = ["en", "zh"] + [f"x{i}" for i in range(98)]
    lang = {f"<|{c}|>": 50259 + i for i, c in enumerate(langs)}
    return dict(decoder_start_token_id=50258, eos_token_id=50257, bos_token_id=50257, pad_token_id=50257,
                no_timestamps_token_id=50364, prev_sot_token_id=50362, is_multilingual=True, lang_to_id=lang,
                task_to_id={"translate": 50359, "transcribe": 50360}, suppress_tokens=[1, 2, 7, 8, 9, 10, 50257, 50361],
                begin_suppress_tokens=[220, 50257], max_initial_timestamp_index=50, max_length=448)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def seed_weights(net, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if "layer_norm" in name:
                p.fill_(1.0 if name.endswith("weight") else 0.0)
            elif name.endswith("bias"):
                p.normal_(0.0, 0.02, generator=g)
            elif "embed" in name:
                p.normal_(0.0, 0.02, generator=g)
            else:
                p.normal_(0.0, 1.0 / math.sqrt(p[0].numel()), generator=g)


def clips(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        secs = rng.uniform(2.0, 12.0)
        t = np.arange(int(secs * 32000)) / 32000
        x = 0.2 * np.sin(2 * np.pi * rng.uniform(100, 400) * t) + 0.05 * rng.standard_normal(t.size)
        out.append(x.astype(np.float32))
    return out


def encoder_flops(c):
    d, M, f, T = c["d_model"], c["num_mel_bins"], c["encoder_ffn_dim"], 1500
    conv = 2 * 3000 * M * 3 * d + 2 * T * d * 3 * d
    layer = 2 * T * d * 3 * d + 4 * T * T * d + 2 * T * d * d + 2 * 2 * T * d * f
    return conv + c["encoder_layers"] * layer


def step_linear_bytes(c, elem):
    """Weight bytes the decode step's Linears read once each: per layer QKV (3 d^2), out, cross-q, cross-out (d^2 each),
    fc1 and fc2 (d * ffn each), and the tied head (V * d)."""
    d, f = c["d_model"], c["decoder_ffn_dim"]
    return elem * (c["decoder_layers"] * (6 * d * d + 2 * d * f) + c["vocab_size"] * d)


HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--compare-clips", type=int, default=16)
    ap.add_argument("--no-compare", action="store_true")
    ap.add_argument("--tokens-per-second", type=float, default=4.0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--long", action="store_true")
    ap.add_argument("--tokens-per-window", type=int, default=120)
    ap.add_argument("--precision", choices=["float16", "bfloat16"], default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_asr needs a GPU")
    if a.long:
        return main_long(a)
    from easevoice_trainer_b200 import asr, lib, normalize_ssl, ops, whisper
    lib.init().evk_set_precise(0)
    dev = torch.device("cuda", 0)
    cfg, gen = dict(whisper.LARGE_V3), generation_config()
    with torch.device(dev):
        net = whisper.WhisperModel(cfg, gen)
    net = net.to(dev).eval()
    seed_weights(net, a.seed)
    sp = net.sp
    xs = sorted(clips(a.clips, a.seed + 1), key=len)
    secs = [x.size / 32000 for x in xs]
    budget = [math.ceil(a.tokens_per_second * s) for s in secs]
    # equal batches: the largest divisor of the clip count within the memory budget's batch size (8 for 256 clips), so one
    # captured decode state serves every batch
    nb = max(k for k in range(1, asr.clips_per_batch(cfg) + 1) if len(xs) % k == 0)
    taps = torch.from_numpy(normalize_ssl.resample_taps()[1]).to(dev)
    batches = [list(range(i, min(i + nb, len(xs)))) for i in range(0, len(xs), nb)]

    def feats_of(idx):
        rows = [ops.resample_poly(torch.from_numpy(xs[i]).to(dev)[None], taps, 1, 2, 64, (xs[i].size + 1) // 2)[0] for i in idx]
        w = torch.zeros(len(rows), max(r.numel() for r in rows), device=dev)
        for j, r in enumerate(rows):
            w[j, :r.numel()] = r
        return net.features(w, [r.numel() for r in rows])

    def run(idx, timing=None):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        f = feats_of(idx)
        ev[1].record()
        enc = net.encode(f)
        ev[2].record()
        out = net.transcribe_features(f, language="en", max_new_tokens=max(budget[i] for i in idx), check_every=1 << 30, enc=enc)
        ev[3].record()
        if timing is not None:
            torch.cuda.synchronize()
            timing["front"] += ev[0].elapsed_time(ev[1])
            timing["encoder"] += ev[1].elapsed_time(ev[2])
            timing["decode"] += ev[2].elapsed_time(ev[3])
        return out

    @torch.no_grad()
    def measure():
        for bt in batches:                                          # warm up: capture the step of every token budget
            run(bt)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        timing = dict(front=0.0, encoder=0.0, decode=0.0)
        t0 = time.perf_counter()
        toks = []
        for bt in batches:
            toks += run(bt, timing)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        # split of the decode: cross K/V of one batch by events, and the beam step's share of one profiled eager step
        bt = batches[-1]
        enc = net.encode(feats_of(bt))
        _, st = net._graph(len(bt), 5, dev, max(budget[i] for i in bt))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        net.cross_kv(enc, st["ckv"])
        e1.record()
        torch.cuda.synchronize()
        ckv_ms_batch = e0.elapsed_time(e1)
        ops.profile_begin()
        lg = net._forward_rows(st)
        ops.whisper_beam_step(lg, st, 5, net._layout(3, 224))
        prof = ops.profile_end()
        step_ms = sum(v["ms"] for v in prof.values())
        lin_ms = sum(v["ms"] for k, v in prof.items() if k.startswith(("evk_gconv_fwd", "evk_linear")))
        beam_ms = prof.get("evk_whisper_beam_step", {}).get("ms", 0.0)
        ckv_ms = ckv_ms_batch * len(xs) / len(bt)
        elem = 4 if net.compute_type is None else 2
        return dict(metric="whisper large-v3-shaped transcription audio-seconds/s", card=card(), clips=len(xs),
                    audio_s=sum(secs), tokens_per_second_of_audio=a.tokens_per_second, clips_per_batch=nb,
                    value=sum(secs) / wall, wall_s=wall, peak_mem_gib=peak,
                    device_ms=dict(front_end=timing["front"], encoder=timing["encoder"], cross_kv_est=ckv_ms,
                                   decode_incl_cross_kv=timing["decode"], beam_step_share_of_eager_step=beam_ms / step_ms if step_ms else None,
                                   eager_step_by_call={k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[:8]}),
                    encoder_tflops=encoder_flops(cfg) * len(xs) / (timing["encoder"] * 1e-3) / 1e12,
                    generated_tokens=sum(len(t["tokens"]) for t in toks), compute_type=str(net.compute_type),
                    eager_step_ms=step_ms, step_linear_ms=lin_ms, step_linear_share=lin_ms / step_ms if step_ms else None,
                    step_linear_floor_ms=step_linear_bytes(cfg, elem) / HBM_BYTES_PER_S * 1e3)

    if a.precision is None:
        res = measure()
    else:
        h16 = asr.compute_dtype(a.precision)
        arms = []
        for dt in (None, h16, None, h16):
            net.set_compute_type(dt)
            arms.append(measure())
        res = dict(arms[-1], arms=arms)
    if not a.no_compare:
        res["transformers"] = compare(net, cfg, gen, xs[:a.compare_clips], budget[:a.compare_clips], nb, feats_of, dev)
    print(json.dumps(res))


def main_long(a):
    from easevoice_trainer_b200 import asr, lib, whisper
    lib.init().evk_set_precise(0)
    dev = torch.device("cuda", 0)
    cfg, gen = dict(whisper.LARGE_V3), generation_config()
    with torch.device(dev):
        net = whisper.WhisperModel(cfg, gen)
    net = net.to(dev).eval()
    seed_weights(net, a.seed)
    n = a.clips if a.clips != 256 else 8
    rng = np.random.default_rng(a.seed + 1)
    xs = []
    for _ in range(n):
        t = np.arange(int(rng.uniform(40.0, 300.0) * 16000)) / 16000
        xs.append((0.2 * np.sin(2 * np.pi * rng.uniform(100, 400) * t) + 0.05 * rng.standard_normal(t.size)).astype(np.float32))
    lens = [x.size for x in xs]
    frames = [m // 160 for m in lens]
    nb = asr.clips_per_batch(cfg, asr.DEFAULT_MEMORY_BUDGET * (1 - asr.LONG_POOL_SHARE))
    tpw = a.tokens_per_window
    timing = dict(encoder=0.0, decode=0.0)
    encode, decode = net.encode, net._decode

    def timed(key, fn):
        def run(*args, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*args, **kw)
            e1.record()
            torch.cuda.synchronize()
            timing[key] += e0.elapsed_time(e1)
            return out
        return run

    def wav():
        w = torch.zeros(n, max(lens), device=dev)
        for i, x in enumerate(xs):
            w[i, :x.size] = torch.from_numpy(x).to(dev)
        return w

    with torch.no_grad():
        w = wav()
        lm = net.features_long(w[:2], lens[:2])                      # warm up: front end, encoder, the pool's graph
        net._graph(min(nb, n), 5, dev, tpw, True)
        net.encode(torch.zeros(1, 3000, cfg["num_mel_bins"], device=dev))
        del lm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        net.encode, net._decode = timed("encoder", encode), timed("decode", decode)
        t0 = time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lm = net.features_long(wav(), lens)
        e1.record()
        res = net.transcribe_long(lm, frames, language="en", clips_per_batch=nb, max_new_tokens=tpw, check_every=1 << 30)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        net.encode, net._decode = encode, decode
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
    audio = sum(lens) / 16000
    out = dict(metric="whisper large-v3-shaped long-form transcription audio-seconds/s", card=card(), clips=n, audio_s=audio,
               clip_s=[round(m / 16000, 1) for m in lens], windows=sum(len(o["windows"]) for o in res), clips_per_batch=min(nb, n),
               tokens_per_window=tpw, value=audio / wall, wall_s=wall, peak_mem_gib=peak,
               device_ms=dict(front_end=e0.elapsed_time(e1), encoder=timing["encoder"], decode_incl_cross_kv=timing["decode"]))
    if not a.no_compare:
        out["transformers"] = compare_long(net, cfg, gen, lm, frames, audio, min(nb, n), tpw, dev)
    print(json.dumps(out))


def compare_long(net, cfg, gen, lm, frames, audio, nb, tpw, dev):
    """transformers' long-form generate on the same whole-clip features, batches of nb clips with an attention_mask."""
    from transformers import GenerationConfig, WhisperConfig, WhisperForConditionalGeneration
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    hc = WhisperConfig(**cfg, decoder_start_token_id=50258, eos_token_id=50257, pad_token_id=50257, bos_token_id=50257,
                       activation_function="gelu", scale_embedding=False, tie_word_embeddings=True)
    with torch.device(dev):
        ref = WhisperForConditionalGeneration(hc)
    missing, unexpected = ref.load_state_dict({k: v.detach() for k, v in net.state_dict().items()}, strict=False)
    assert not unexpected and set(missing) <= {"proj_out.weight"}, (missing, unexpected)
    ref.tie_weights()
    ref.eval().to(dev)
    feats = lm.transpose(1, 2).contiguous()
    mask = (torch.arange(feats.shape[2], device=dev)[None] < torch.tensor(frames, device=dev)[:, None]).long()
    kw = dict(num_beams=5, return_timestamps=True, task="transcribe", language="en", temperature=0.0, logprob_threshold=-1.0,
              no_speech_threshold=0.6, condition_on_prev_tokens=False)
    out = {}
    for dt in (torch.float32, torch.float16):
        m = ref.to(dt)
        m.generation_config = GenerationConfig(**gen)
        with torch.no_grad():
            m.generate(feats[:1, :, :3000].to(dt), num_beams=5, return_timestamps=True, task="transcribe", language="en",
                       max_new_tokens=4)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(0, feats.shape[0], nb):
                T = max(frames[i:i + nb])
                m.generate(feats[i:i + nb, :, :T].to(dt), attention_mask=mask[i:i + nb, :T], max_new_tokens=tpw, **kw)
            torch.cuda.synchronize()
        out[f"{str(dt).split('.')[-1]}_batched"] = dict(audio_s_per_s=audio / (time.perf_counter() - t0), clips=feats.shape[0])
    return out


def compare(net, cfg, gen, xs, budget, nb, feats_of, dev):
    """transformers' generate(num_beams=5, return_timestamps=True) with the same weights and features: fp32 with TF32 allowed
    and fp16, one clip per call and in batches of nb."""
    from transformers import GenerationConfig, WhisperConfig, WhisperForConditionalGeneration
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    hc = WhisperConfig(**cfg, decoder_start_token_id=50258, eos_token_id=50257, pad_token_id=50257, bos_token_id=50257,
                       activation_function="gelu", scale_embedding=False, tie_word_embeddings=True)
    with torch.device(dev):
        ref = WhisperForConditionalGeneration(hc)
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not unexpected and set(missing) <= {"proj_out.weight"}, (missing, unexpected)
    ref.tie_weights()
    ref.eval().to(dev)
    audio = sum(x.size for x in xs) / 32000
    with torch.no_grad():
        feats = feats_of(list(range(len(xs)))).transpose(1, 2).contiguous()
    out = {}
    for dt in (torch.float32, torch.float16):
        m = ref.to(dt)
        m.generation_config = GenerationConfig(**gen)
        for name, size in (("one_clip_per_call", 1), ("batched", nb)):
            def go():
                for i in range(0, len(xs), size):
                    m.generate(feats[i:i + size].to(dt), num_beams=5, return_timestamps=True, task="transcribe", language="en",
                               max_new_tokens=max(budget[i:i + size]))
            with torch.no_grad():
                m.generate(feats[:1].to(dt), num_beams=5, return_timestamps=True, task="transcribe", language="en",
                           max_new_tokens=4)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                go()
                torch.cuda.synchronize()
            out[f"{str(dt).split('.')[-1]}_{name}"] = dict(audio_s_per_s=audio / (time.perf_counter() - t0), clips=len(xs))
    return out


if __name__ == "__main__":
    main()
