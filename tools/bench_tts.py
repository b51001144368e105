#!/usr/bin/env python
"""Time tts.run, the whole synthesis call, on seeded full-size models: the 24-layer GPT, the shipped s2 config and
HuBERT-base.  20 sentences of 20-60 phonemes, a 150-token prompt (a 5.4 s clip), batch_size 8, top_k 15, 300-token caps.

Prints one JSON line: the call from its start to the int16 array (synchronised), split into prompt preparation
(set_ref_audio), AR decoding (infer_panel), vocoding (decode) and assembly plus copy (audio_postprocess), each from CUDA
events around the wrapped calls; and the assembly (evk_fragment_int16 + one copy) against the reference's host
audio_postprocess (per-fragment max, division, .cpu().numpy(), host concatenation and cast) on the same vocoder outputs,
alternated in one process.  The card name and power limit are read in the same call.

--precision float16|bfloat16: every round runs the call once with the fp32 and once with the 16-bit compute type of the
GPT's AR decoding (Text2SemanticDecoder.set_compute_type, what enable_half_precision selects), alternated; each call also
reports its peak allocated memory.

Usage:  python tools/bench_tts.py [--reps 3] [--precision float16|bfloat16]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gpt_oracle, hubert_oracle, s2_oracle, tts_oracle as to  # noqa: E402

DEV = torch.device("cuda", 0)


def models():
    from easevoice_trainer_b200 import configs, hubert
    from easevoice_trainer_b200 import models as s2
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    m = dict(gpt_oracle.GPT_MODEL)
    t2s = Text2SemanticDecoder({"model": m})
    t2s.load_state_dict(gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), 14))
    hps = configs.load_s2_config()
    vits = s2.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                             n_speakers=hps["data"]["n_speakers"], **hps["model"])
    vits.load_state_dict(s2_oracle.init_params(s2_oracle.generator_param_spec(), 1234))
    hub = hubert.HubertModel({})
    hub.load_state_dict(hubert_oracle.init_params(hubert_oracle.param_spec(), 42))
    return t2s.to(DEV).eval(), vits.to(DEV).eval(), types.SimpleNamespace(model=hub.to(DEV).eval()), hps


class Preprocessor:
    def __init__(self, n, seed):
        g = torch.Generator().manual_seed(seed)
        self.sent = []
        for _ in range(n):
            x = int(torch.randint(20, 61, (1,), generator=g))
            self.sent.append({"phones": torch.randint(0, 732, (x,), generator=g).tolist(),
                              "bert_features": torch.randn(1024, x, generator=g), "norm_text": "t" * x})
        x = 30
        self.prompt = ([int(v) for v in torch.randint(0, 732, (x,), generator=g)], torch.randn(1024, x, generator=g), "p" * x)

    def preprocess(self, text, lang, method):
        return [dict(s) for s in self.sent]

    def segment_and_extract_feature_for_text(self, text, lang):
        return list(self.prompt[0]), self.prompt[1].clone(), self.prompt[2]


class Caller:
    """the caller's TTS object around this library's models"""

    def __init__(self, tts, t2s, vits, hub, hps, clip32, clip16):
        self._tts, self.clip32, self.clip16 = tts, clip32, clip16
        self.t2s_model, self.vits_model, self.cnhuhbert_model = types.SimpleNamespace(model=t2s), vits, hub
        d = hps["data"]
        self.configs = types.SimpleNamespace(device=DEV, sampling_rate=d["sampling_rate"], filter_length=d["filter_length"],
                                             hop_length=d["hop_length"], win_length=d["win_length"], hz=50, max_sec=6,
                                             languages=to.LANGS, t2s_weights_path="", vits_weights_path="")
        self.text_preprocessor = Preprocessor(20, 5)
        self.reset()

    def reset(self):
        self.prompt_cache = {"ref_audio_path": None, "prompt_semantic": None, "refer_spec": [], "prompt_text": None,
                             "prompt_lang": None, "phones": None, "bert_features": None, "norm_text": None, "aux_ref_audio_paths": []}

    def set_ref_audio(self, path):
        c = self.configs
        self.prompt_cache["prompt_semantic"] = self._tts.prompt_semantic(self.clip16, self.cnhuhbert_model, self.vits_model,
                                                                        c.sampling_rate)
        self.prompt_cache["refer_spec"] = [self._get_ref_spec(path)]
        self.prompt_cache["ref_audio_path"] = path

    def _get_ref_spec(self, path):
        c = self.configs
        return self._tts.ref_spec(self.clip32, c.filter_length, c.sampling_rate, c.hop_length, c.win_length, c.device)


def reference_postprocess(audio, sr, batch_index_list, fragment_interval):
    """the reference's audio_postprocess loop (tts.py:886-907) on device fragments"""
    zero_wav = torch.zeros(int(sr * fragment_interval), dtype=torch.float32, device=DEV)
    out = [[None] * len(b) for b in audio]
    for i, batch in enumerate(audio):
        for j, frag in enumerate(batch):
            frag = frag.clone()
            m = torch.abs(frag).max()
            if m > 1:
                frag /= m
            out[i][j] = torch.cat([frag, zero_wav], dim=0).cpu().numpy()
    flat = to.recovery_order(out, batch_index_list)
    return sr, (np.concatenate(flat, 0) * 32768).astype(np.int16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", choices=["float16", "bfloat16"], default=None)
    args = ap.parse_args()
    from easevoice_trainer_b200 import lib, tts
    lib.init()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    t2s, vits, hub, hps = models()
    g = torch.Generator().manual_seed(3)
    n16 = 150 * 2 * 320 - int(hps["data"]["sampling_rate"] * 0.3)          # 150 prompt tokens with the 0.6 s padding
    t = torch.arange(2 * n16) / 32000.0
    clip32 = (0.4 * torch.sin(2 * np.pi * 150 * t) + 0.05 * torch.randn(2 * n16, generator=g)).float().numpy()
    clip16 = clip32[::2].copy()
    caller = Caller(tts, t2s, vits, hub, hps, clip32, clip16)

    phases = {"prompt": [], "ar": [], "vocode": [], "assemble": []}

    def timed(key, fn):
        def wrap(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            phases[key].append((e0, e1))
            return out
        return wrap
    caller.set_ref_audio = timed("prompt", caller.set_ref_audio)
    t2s.infer_panel_batch_infer = timed("ar", type(t2s).infer_panel_batch_infer.__get__(t2s))
    vits.decode = timed("vocode", type(vits).decode.__get__(vits))
    keep = {}
    post = tts.audio_postprocess

    def spy_post(audio, *a):
        keep["audio"], keep["args"] = audio, a
        return post(audio, *a)
    tts.audio_postprocess = timed("assemble", spy_post)

    with tempfile.NamedTemporaryFile(suffix=".wav") as f:
        inputs = dict(text="t", text_lang="zh", ref_audio_path=f.name, prompt_text="p", prompt_lang="zh", top_k=15, batch_size=8,
                      seed=7, fragment_interval=0.3)
        arms = [None] if args.precision is None else [None, getattr(torch, args.precision)]
        per_arm = {str(dt): [] for dt in arms}
        for rep in range(args.reps + 1):                                    # the first round warms every shape up
            for dt in arms:
                t2s.set_compute_type(dt)
                for v in phases.values():
                    v.clear()
                caller.reset()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                sr, wav = next(tts.run(caller, inputs))
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if rep:
                    per_arm[str(dt)].append(dict(wall_ms=wall * 1e3, samples=int(wav.shape[0]),
                                                 peak_mem_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
                                                 **{k + "_ms": sum(a.elapsed_time(b) for a, b in v) for k, v in phases.items()}))
        calls = per_arm["None"]
    tts.audio_postprocess = post
    audio, (sr, bil, speed, split, interval) = keep["audio"], keep["args"]
    ours, ref = [], []
    for _ in range(10):                                                     # alternated, same device fragments
        torch.cuda.synchronize(); t0 = time.perf_counter()
        _, a = post(audio, sr, bil, speed, split, interval)
        ours.append(time.perf_counter() - t0)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        _, b = reference_postprocess(audio, sr, bil, interval)
        ref.append(time.perf_counter() - t0)
    assert np.array_equal(a, b), "assembly differs from the reference's host loop"
    med = lambda v: float(np.median(v))                                     # noqa: E731
    print(json.dumps({"card": card, "sentences": 20, "fragments": sum(len(x) for x in audio), "audio_s": calls[-1]["samples"] / sr,
                      "calls": calls, "median_wall_ms": med([c["wall_ms"] for c in calls]),
                      "assembly_ms": med(ours) * 1e3, "reference_host_postprocess_ms": med(ref) * 1e3,
                      **({} if args.precision is None else {"arms": {k: dict(calls=v, median_wall_ms=med([c["wall_ms"] for c in v]),
                                                                            median_ar_ms=med([c["ar_ms"] for c in v]))
                                                                     for k, v in per_arm.items()}})}))


if __name__ == "__main__":
    main()
