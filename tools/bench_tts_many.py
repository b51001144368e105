#!/usr/bin/env python
"""Time tts.run_many against the same requests through tts.run one after another, on seeded full-size models: the 24-layer
GPT and the shipped s2 config (HuBERT-base for the prompt tokens).  16 requests of 1-3 sentences (20-60 phonemes), each with
its own seeded reference clip of 3-10 s, its own seed and sampling settings, batch_size 4, 300-token caps.

The two arms alternate in one process, after one warm-up call of each.  Prints one JSON line: per arm the wall time of the
whole call (synchronised), the device time of AR decoding (decode_groups / infer_panel_batch_infer), vocoding (decode,
decode_batch) and
int16 assembly (evk_fragment_int16 calls) from CUDA events around the wrapped calls, and the peak allocated memory; and the
card name and power limit, read in the same call.

--precision float16|bfloat16: run_many alone, with the fp32 and the 16-bit compute type of the GPT's AR decoding
(Text2SemanticDecoder.set_compute_type) as the two alternated arms instead.

Usage:  python tools/bench_tts_many.py [--reps 3] [--precision float16|bfloat16]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tts import Caller, models  # noqa: E402

DEV = torch.device("cuda", 0)
N_REQ = 16


class Preprocessor:
    """per request: 1-3 seeded sentences (keyed by the request's text) and a 30-phoneme prompt"""

    def __init__(self):
        g = torch.Generator().manual_seed(9)
        self.sent = {}
        for r in range(N_REQ):
            out = []
            for _ in range(int(torch.randint(1, 4, (1,), generator=g))):
                x = int(torch.randint(20, 61, (1,), generator=g))
                out.append({"phones": torch.randint(0, 732, (x,), generator=g).tolist(),
                            "bert_features": torch.randn(1024, x, generator=g), "norm_text": "t" * x})
            self.sent[f"r{r}"] = out
        self.prompt = ([int(v) for v in torch.randint(0, 732, (30,), generator=g)], torch.randn(1024, 30, generator=g), "p" * 30)

    def preprocess(self, text, lang, method):
        return [dict(s) for s in self.sent[text]]

    def segment_and_extract_feature_for_text(self, text, lang):
        return list(self.prompt[0]), self.prompt[1].clone(), self.prompt[2]


class ManyCaller(Caller):
    """Caller with one seeded clip per reference path"""

    def __init__(self, tts, t2s, vits, hub, hps, clips):
        super().__init__(tts, t2s, vits, hub, hps, None, None)
        self.clips = clips
        self.text_preprocessor = Preprocessor()

    def set_ref_audio(self, path):
        self.clip32, self.clip16 = self.clips[path]
        super().set_ref_audio(path)

    def _get_ref_spec(self, path):
        self.clip32 = self.clips[path][0]
        return super()._get_ref_spec(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", choices=["float16", "bfloat16"], default=None)
    args = ap.parse_args()
    from easevoice_trainer_b200 import lib, ops, tts
    lib.init()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    t2s, vits, hub, hps = models()
    g = torch.Generator().manual_seed(3)
    with tempfile.TemporaryDirectory() as d:
        clips, inputs = {}, []
        for r in range(N_REQ):
            n = int((3.2 + 6.5 * float(torch.rand(1, generator=g))) * 32000)
            t = torch.arange(n) / 32000.0
            x = (0.4 * torch.sin(2 * np.pi * (100 + 100 * float(torch.rand(1, generator=g))) * t)
                 + 0.05 * torch.randn(n, generator=g)).float().numpy()
            path = os.path.join(d, f"clip{r}.wav")
            open(path, "wb").close()
            clips[path] = (x, x[::2].copy())
            inputs.append(dict(text=f"r{r}", text_lang="zh", ref_audio_path=path, prompt_text="p", prompt_lang="zh",
                               top_k=[5, 15, 30][r % 3], top_p=[1.0, 0.9][r % 2], temperature=[1.0, 0.8][(r // 2) % 2],
                               repetition_penalty=1.35, batch_size=4, seed=100 + r, fragment_interval=0.3))
        caller = ManyCaller(tts, t2s, vits, hub, hps, clips)

        phases = {"ar": [], "vocode": [], "assemble": []}

        def timed(key, fn):
            def wrap(*a, **k):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn(*a, **k)
                e1.record()
                phases[key].append((e0, e1))
                return out
            return wrap
        t2s.infer_panel_batch_infer = timed("ar", type(t2s).infer_panel_batch_infer.__get__(t2s))
        t2s.decode_groups = timed("ar", type(t2s).decode_groups.__get__(t2s))
        vits.decode = timed("vocode", type(vits).decode.__get__(vits))
        vits.decode_batch = timed("vocode", type(vits).decode_batch.__get__(vits))
        frag = ops.fragment_int16
        ops.fragment_int16 = timed("assemble", frag)

        def arm_many():
            results, errors = tts.run_many(caller, inputs)
            assert not errors, errors
            return results

        def arm_loop():
            return [next(tts.run(caller, inp)) for inp in inputs]
        if args.precision is None:
            arms = (("run_many", arm_many), ("run_loop", arm_loop))
        else:
            def typed(dt):
                def arm():
                    t2s.set_compute_type(dt)
                    return arm_many()
                return arm
            arms = (("run_many", typed(None)), ("run_many_" + args.precision, typed(getattr(torch, args.precision))))
        out = {name: [] for name, _ in arms}
        samples = {}
        for rep in range(args.reps + 1):                                    # the first round warms every shape up
            for name, fn in arms:
                for v in phases.values():
                    v.clear()
                caller.reset()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                res = fn()
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                samples[name] = sum(int(a.shape[0]) for _, a in res)
                if rep:
                    out[name].append(dict(wall_ms=wall * 1e3, peak_mem_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
                                          **{k + "_ms": sum(a.elapsed_time(b) for a, b in v) for k, v in phases.items()}))
        ops.fragment_int16 = frag
    med = lambda v: float(np.median(v))                                     # noqa: E731
    sent = sum(len(v) for v in caller.text_preprocessor.sent.values())
    print(json.dumps({"card": card, "requests": N_REQ, "sentences": sent, "audio_s": {k: v / 32000 for k, v in samples.items()},
                      **out, "median_wall_ms": {k: med([c["wall_ms"] for c in v]) for k, v in out.items()},
                      "median_ar_ms": {k: med([c["ar_ms"] for c in v]) for k, v in out.items()},
                      # run_loop over run_many; with --precision, fp32 over 16-bit
                      "speedup": (lambda a, b: med([c["wall_ms"] for c in out[a]]) / med([c["wall_ms"] for c in out[b]]))(
                          *(("run_loop", "run_many") if args.precision is None else ("run_many", arms[1][0])))}))


if __name__ == "__main__":
    main()
