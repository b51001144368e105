#!/usr/bin/env python
"""Pin the long-form seek loop of the Whisper oracle (whisper_long_oracle.transcribe_long) against transformers' long-form
`generate` on the CPU and write tests/golden/asr_long.pt.

transformers runs `generate(num_beams=5, return_timestamps=True, task="transcribe", max_new_tokens=224, temperature=0.0,
logprob_threshold=-1.0, no_speech_threshold=0.6, condition_on_prev_tokens=False)` on the oracle's whole-clip features
(log_mel, [n_mels, frames]): each clip alone, and the clips together, padded with zeros and with an `attention_mask`.  The
pin checks, per clip:
  1. alone and batched give the same tokens and the same seeks (the seek at each window, from `monitor_progress`);
  2. the oracle's seeks and kept tokens equal them, and its language equals `detect_language` on the first window;
  3. the oracle's avg_logprob, no_speech_prob and skip flag per window equal those `_need_fallback` computed.

The model is pin_asr's m80_d2 with three changes that make random weights exercise the seek rules: the timestamp rows of
the tied embedding and the <|nospeech|> row get the direction of the decoder's final LayerNorm bias (timestamps are
predicted, and some windows have a high no-speech probability), and <|nospeech|> is suppressed, as openai-whisper
suppresses it.  The goldens cover windows whose segments end at a timestamp pair (seek lands mid-window), windows without a
pair (seek moves by the window), skipped no-speech windows, short last windows, and detected and forced languages.

Usage:  python oracle/pin_asr_long.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pin_asr as PIN  # noqa: E402
from oracle import whisper_long_oracle as L  # noqa: E402
from oracle import whisper_oracle as W  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "asr_long.pt")
CASE = dict(cfg=PIN.CASES["m80_d2"]["cfg"], seed=3, eot_gain=6.0, ts_gain=8.0, nospeech_gain=40.0)
# clips: (seed, seconds, silent span in seconds or None)
CLIPS = [(70, 75.3, (31.0, 62.0)), (75, 52.9, (20.0, 25.0))]
LANGS = (None, "de")


def generation_config():
    gen = PIN.generation_config()
    return dict(gen, suppress_tokens=gen["suppress_tokens"] + [gen["no_timestamps_token_id"] - 1])


def make_state_dict(c=CASE):
    cfg = PIN.full_cfg(c["cfg"])
    sd = PIN.make_state_dict(cfg, c["seed"], c["eot_gain"])
    sp = W.special_tokens(generation_config())
    E, b = sd["model.decoder.embed_tokens.weight"], sd["model.decoder.layer_norm.bias"]
    E[sp["ts_begin"]:] += c["ts_gain"] * b / b.norm()
    E[sp["nospeech"]] = c["nospeech_gain"] * b / b.norm()
    return sd


def clip(seed, secs, silence):
    x = PIN.clip(seed, secs)
    if silence is not None:
        x[int(silence[0] * W.SR):int(silence[1] * W.SR)] = 0.0
    return x


def endings(res, sp):
    """The seek cases a clip's windows reach: pair (seek moved to a timestamp pair inside the window), single (the
    hypothesis ends in one timestamp after text), skipped, short_last (a last window under 3000 frames)."""
    out = set()
    for w in res["windows"]:
        seq = w["tokens"][:-1] if w["tokens"] and w["tokens"][-1] == sp["eot"] else w["tokens"]
        if w["skipped"]:
            out.add("skipped")
        elif L.retrieve_segment(seq, sp["ts_begin"], w["n_frames"])[1] < w["n_frames"]:
            out.add("pair")
        elif len(seq) >= 2 and seq[-2] < sp["ts_begin"] <= seq[-1]:
            out.add("single")
    if res["windows"][-1]["n_frames"] < W.N_FRAMES:
        out.add("short_last")
    return out


def main():
    from transformers import GenerationConfig, WhisperConfig, WhisperForConditionalGeneration
    from transformers.models.whisper import generation_whisper as GW
    torch.set_grad_enabled(False)
    gen = generation_config()
    sp = W.special_tokens(gen)
    cfg = PIN.full_cfg(CASE["cfg"])
    sd = make_state_dict()
    hc = WhisperConfig(**cfg, decoder_start_token_id=sp["sot"], eos_token_id=sp["eot"], pad_token_id=sp["eot"],
                       bos_token_id=sp["eot"], activation_function="gelu", scale_embedding=False, tie_word_embeddings=True)
    net = WhisperForConditionalGeneration(hc).double().eval()
    missing, unexpected = net.load_state_dict({k: v.double() for k, v in sd.items()}, strict=False)
    assert not unexpected and set(missing) <= {"proj_out.weight"}, (missing, unexpected)
    net.tie_weights()
    net.generation_config = GenerationConfig(**gen)

    # what _need_fallback decided per window, in call order: (avg_logprob, no_speech_prob, should_skip)
    seen = []
    need_fallback = GW.WhisperGenerationMixin._need_fallback

    def spy(self, seq, outs, i, procs, gcfg, V, temperature):
        r = need_fallback(self, seq, outs, i, procs, gcfg, V, temperature)
        alp = float(self._retrieve_avg_logprobs(outs[i]["scores"], seq, temperature))
        nsp = float(GW._get_attr_from_logit_processors(procs, GW.WhisperNoSpeechDetection, "no_speech_prob")[i])
        seen.append((alp, nsp, bool(r[1])))
        return r

    GW.WhisperGenerationMixin._need_fallback = spy

    waves = [clip(*c) for c in CLIPS]
    lms = [W.log_mel(x, cfg["num_mel_bins"]) for x in waves]
    frames = [lm.shape[0] for lm in lms]

    def generate(feats, mask, lang):
        trace = []
        kw = dict(num_beams=5, return_timestamps=True, task="transcribe", max_new_tokens=224, temperature=0.0,
                  logprob_threshold=-1.0, no_speech_threshold=0.6, condition_on_prev_tokens=False, return_segments=True,
                  monitor_progress=lambda t: trace.append(t[:, 0].tolist()))
        if lang is not None:
            kw["language"] = lang
        if mask is not None:
            kw["attention_mask"] = mask
        o = net.generate(feats, **kw)
        toks = [[t for s in segs for t in s["tokens"].tolist()] for segs in o["segments"]]
        seeks = [[] for _ in toks]
        for row in trace:
            for i, s in enumerate(row):
                if s < frames_of[i] and (not seeks[i] or seeks[i][-1] != s):
                    seeks[i].append(int(s))
        return toks, seeks

    runs, covered = [], set()
    for lang in LANGS:
        alone, decided = [], []
        for i, lm in enumerate(lms):
            frames_of = [frames[i]]
            seen.clear()
            t, s = generate(lm.T[None].contiguous(), None, lang)
            alone.append((t[0], s[0]))
            decided.append(list(seen))
        T = max(frames)
        feats = torch.zeros(len(lms), cfg["num_mel_bins"], T, dtype=torch.float64)
        mask = torch.zeros(len(lms), T, dtype=torch.long)
        for i, lm in enumerate(lms):
            feats[i, :, :lm.shape[0]] = lm.T
            mask[i, :lm.shape[0]] = 1
        frames_of = frames
        bt, bs = generate(feats, mask, lang)
        results = []
        for i, x in enumerate(waves):
            assert (bt[i], bs[i]) == alone[i], f"clip {i} lang {lang}: batched {bs[i]} {bt[i]} != alone {alone[i]}"
            o = L.transcribe_long(sd, cfg, sp, x, language=lang)
            seeks = [w["seek"] for w in o["windows"]]
            assert seeks == alone[i][1], f"clip {i} lang {lang}: oracle seeks {seeks} != generate {alone[i][1]}"
            assert o["tokens"] == alone[i][0], f"clip {i} lang {lang}: oracle {o['tokens']} != generate {alone[i][0]}"
            if lang is None:
                lid = int(net.detect_language(input_features=lms[i].T[None, :, :3000].contiguous(), generation_config=net.generation_config)[0])
                assert sp["langs"][o["language"]] == lid, (o["language"], lid)
            assert len(decided[i]) == len(o["windows"])
            for w, (alp, nsp, skip) in zip(o["windows"], decided[i]):
                assert w["skipped"] == skip and abs(w["avg_logprob"] - alp) < 1e-5 and abs(w["no_speech_prob"] - nsp) < 1e-9, \
                    (i, lang, w["seek"], w["avg_logprob"], alp, w["no_speech_prob"], nsp)
            kinds = endings(o, sp)
            covered |= kinds | {"detected" if lang is None else "forced"}
            print(f"lang={lang} clip {i} ({frames[i]} frames) -> {o['language']}: seeks {seeks}, {len(o['tokens'])} tokens, "
                  f"windows {[(w['n_frames'], round(w['avg_logprob'], 3), round(w['no_speech_prob'], 3), w['skipped']) for w in o['windows']]}"
                  f", cases {sorted(kinds)}: identical to generate alone and batched")
            results.append(o)
        runs.append(dict(language=lang, results=results))
    GW.WhisperGenerationMixin._need_fallback = need_fallback
    # a hypothesis ending in one timestamp after text did not occur with these weights; tests/test_cpu_asr_long.py checks
    # that rule on hand-written hypotheses
    want = {"pair", "skipped", "short_last", "detected", "forced"}
    assert want <= covered, f"cases not covered: {want - covered}"
    torch.save(dict(gen=gen, n_text=PIN.N_TEXT, case=dict(CASE, cfg=cfg), clips=CLIPS, frames=frames, runs=runs), GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes")


if __name__ == "__main__":
    main()
