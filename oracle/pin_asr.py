#!/usr/bin/env python
"""Pin the Whisper oracle (oracle/whisper_oracle.py) against transformers on the CPU and write tests/golden/asr.pt.

  1. mel_filters equals transformers' mel_filter_bank(201, n_mels, 0, 8000, 16000, "slaney", "slaney") for 80 and 128 bins;
     log_mel's frames equal WhisperFeatureExtractor's away from the clip's end (the extractor pads the waveform to 30 s,
     the oracle pads the features: the golden keeps both, for the CPU test of where they differ);
  2. with the seeded weights loaded into WhisperForConditionalGeneration in float64, the oracle's encoder output and
     teacher-forced decoder logits match;
  3. process() equals transformers' SuppressTokensAtBegin, SuppressTokens and WhisperTimeStamp processors on random
     log-probs and token histories;
  4. transcribe_clip's tokens equal `generate(num_beams=5, return_timestamps=True, task="transcribe", max_new_tokens=224)`,
     with a given language and with language detection.

The small configs use a 100-token text vocabulary and the multilingual special-token layout written into a generation config
here (eot = 100, four languages, 1501 timestamps: V = 1613).  The goldens keep seeds, configs, teacher-forced logits, token
sequences and scores; weights and clips are regenerated from the seeds by `make_state_dict` and `clip`, and features and
encoder outputs by the oracle, so no test needs transformers.

Usage:  python oracle/pin_asr.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import whisper_oracle as W  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "asr.pt")
N_TEXT = 100
LANGS = ["en", "zh", "de", "ja"]


def generation_config():
    eot = N_TEXT
    sot = eot + 1
    lang = {f"<|{c}|>": sot + 1 + i for i, c in enumerate(LANGS)}
    nxt = sot + 1 + len(LANGS)
    translate, transcribe, startoflm, startofprev, nospeech, notimestamps = range(nxt, nxt + 6)
    return dict(decoder_start_token_id=sot, eos_token_id=eot, bos_token_id=eot, pad_token_id=eot,
                no_timestamps_token_id=notimestamps, prev_sot_token_id=startofprev, is_multilingual=True,
                lang_to_id=lang, task_to_id={"translate": translate, "transcribe": transcribe},
                suppress_tokens=[1, 2, 7, 14, 31, 63, startoflm], begin_suppress_tokens=[5, eot],
                max_initial_timestamp_index=50, max_length=448)


def vocab_size():
    return generation_config()["no_timestamps_token_id"] + 1 + 1501


CASES = {
    # name: model shape, weight seed, clip seconds, eot bias (raises the tied eot row so that some hypotheses finish)
    "m80_d2": dict(cfg=dict(num_mel_bins=80, d_model=128, encoder_layers=2, decoder_layers=2, encoder_attention_heads=2,
                            decoder_attention_heads=2, encoder_ffn_dim=256, decoder_ffn_dim=256), seed=3, secs=[3.1, 7.45], eot_gain=6.0),
    "m128_d4": dict(cfg=dict(num_mel_bins=128, d_model=128, encoder_layers=2, decoder_layers=4, encoder_attention_heads=2,
                             decoder_attention_heads=2, encoder_ffn_dim=256, decoder_ffn_dim=256), seed=4, secs=[5.0], eot_gain=6.0),
}


def full_cfg(c):
    return dict(c, vocab_size=vocab_size(), max_source_positions=1500, max_target_positions=448)


def sinusoids(length, channels):
    inc = np.log(10000) / (channels // 2 - 1)
    inv = torch.exp(-inc * torch.arange(channels // 2, dtype=torch.float64))
    t = torch.arange(length, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.cat([t.sin(), t.cos()], dim=1)


def make_state_dict(cfg, seed, eot_gain=1.0, eot=N_TEXT):
    """Seeded float32 weights: N(0, 1/fan_in) matrices, LayerNorms near identity, sinusoidal encoder positions."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in W.param_spec(cfg):
        if name.endswith("embed_positions.weight") and ".encoder." in name:
            t = sinusoids(*shape).float()
        elif "layer_norm" in name:
            t = (1.0 if name.endswith("weight") else 0.0) + 0.1 * torch.randn(shape, generator=g)
        elif name.endswith("bias"):
            t = 0.05 * torch.randn(shape, generator=g)
        elif name.endswith("embed_tokens.weight") or name.endswith("embed_positions.weight"):
            t = 0.5 * torch.randn(shape, generator=g)
        else:
            fan = int(np.prod(shape[1:]))
            t = torch.randn(shape, generator=g) / fan ** 0.5
        sd[name] = t.float().contiguous()
    sd["model.decoder.embed_tokens.weight"][eot] *= eot_gain
    return sd


def clip(seed, secs):
    g = np.random.default_rng(seed)
    n = int(secs * W.SR)
    t = np.arange(n) / W.SR
    x = 0.3 * np.sin(2 * np.pi * (180 + 40 * g.random()) * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 1.3 * t))
    return (x + 0.05 * g.standard_normal(n)).astype(np.float32)


def main():
    from transformers import GenerationConfig, WhisperConfig, WhisperFeatureExtractor, WhisperForConditionalGeneration
    from transformers.audio_utils import mel_filter_bank
    from transformers.generation.logits_process import (SuppressTokensAtBeginLogitsProcessor, SuppressTokensLogitsProcessor,
                                                        WhisperTimeStampLogitsProcessor)
    torch.set_grad_enabled(False)
    out = dict(gen=generation_config(), n_text=N_TEXT, cases={}, frontend={})
    gen = generation_config()
    sp = W.special_tokens(gen)

    # 1. front end
    for M in (80, 128):
        ref = mel_filter_bank(201, M, 0.0, 8000.0, 16000, norm="slaney", mel_scale="slaney")
        d = np.abs(W.mel_filters(M) - ref).max()
        print(f"mel_filters({M}) max-abs {d:.3e}")
        assert d < 1e-12
        x = clip(100 + M, 4.37)
        fe = WhisperFeatureExtractor(feature_size=M)
        hf = torch.as_tensor(fe(x, sampling_rate=16000, return_tensors="np")["input_features"][0]).T      # [3000, M]
        ours = W.features(x, M)
        T = W.num_frames(x.size)
        inner = T - 3
        # the extractor's max runs over the zero-padded tail too; away from the clip's end both see the same samples
        d = (hf[:inner] - ours[:inner]).abs().max().item()
        print(f"features({M}) frames < {inner}: max-abs vs WhisperFeatureExtractor {d:.3e}")
        assert d < 1e-5
        # the waveform is regenerated from (seed, secs) by clip(); of the extractor's features the clip's frames, 16 after
        # them and the last are kept
        out["frontend"][M] = dict(seed=100 + M, secs=4.37, n_frames=T, hf_head=hf[:T + 16].float().clone(), hf_last=hf[-1].float().clone())

    # 3. processors on random log-probs
    V = vocab_size()
    g = torch.Generator().manual_seed(9)
    tb = sp["ts_begin"]
    proc_cases = []
    for hist_len in (0, 1, 2, 5):
        R = 6
        lp = torch.log_softmax(3 * torch.randn(R, V, generator=g), -1)
        hists = []
        for r in range(R):
            h = []
            for _ in range(hist_len):
                h.append(int(torch.randint(0, N_TEXT, (1,), generator=g)) if torch.rand(1, generator=g) < 0.5
                         else tb + int(torch.randint(0, 60, (1,), generator=g)))
            hists.append(h)
        prompt = [sp["sot"], sp["langs"]["en"], sp["transcribe"]]
        ids = torch.tensor([prompt + h for h in hists])
        gcfg = GenerationConfig(**gen)
        ref = lp.clone()
        for pr in (SuppressTokensAtBeginLogitsProcessor(gen["begin_suppress_tokens"], 3),
                   SuppressTokensLogitsProcessor(gen["suppress_tokens"]), WhisperTimeStampLogitsProcessor(gcfg, begin_index=3)):
            ref = pr(ids, ref)
        ours = W.process(lp, hists, sp)
        assert torch.equal(torch.isinf(ref), torch.isinf(ours)) and torch.equal(ref[~torch.isinf(ref)], ours[~torch.isinf(ours)])
        proc_cases.append(dict(lp=lp, hists=hists, out=ours))
    print("processors: identical on", len(proc_cases), "batches")
    out["processors"] = proc_cases

    # 2. and 4. network and generate
    for name, c in CASES.items():
        cfg = full_cfg(c["cfg"])
        sd = make_state_dict(cfg, c["seed"], c["eot_gain"])
        hc = WhisperConfig(**cfg, decoder_start_token_id=sp["sot"], eos_token_id=sp["eot"], pad_token_id=sp["eot"],
                           bos_token_id=sp["eot"], activation_function="gelu", scale_embedding=False, tie_word_embeddings=True)
        net = WhisperForConditionalGeneration(hc).double().eval()
        missing, unexpected = net.load_state_dict({k: v.double() for k, v in sd.items()}, strict=False)
        assert not unexpected and set(missing) <= {"proj_out.weight"}, (missing, unexpected)
        net.tie_weights()
        net.generation_config = GenerationConfig(**gen)
        M = cfg["num_mel_bins"]
        waves = [clip(c["seed"] * 10 + i, s) for i, s in enumerate(c["secs"])]
        feats = torch.stack([W.features(x, M) for x in waves])
        enc = W.encode(sd, feats, cfg)
        enc_hf = net.model.encoder(feats.transpose(1, 2)).last_hidden_state
        print(f"{name}: encoder max-abs {(enc - enc_hf).abs().max():.3e}")
        assert (enc - enc_hf).abs().max() < 1e-9
        toks = torch.tensor([[sp["sot"], sp["langs"]["de"], sp["transcribe"], tb + 3, 17, 42, 5, tb + 20]] * len(waves))
        lg = W.decode_logits(sd, enc, toks, cfg)
        lg_hf = net(encoder_outputs=(enc_hf,), decoder_input_ids=toks).logits
        print(f"{name}: decoder logits max-abs {(lg - lg_hf).abs().max():.3e}")
        assert (lg - lg_hf).abs().max() < 1e-9
        runs = []
        for lang in ("zh", None):
            kw = dict(num_beams=5, return_timestamps=True, task="transcribe", max_new_tokens=224)
            if lang is not None:
                kw["language"] = lang
            res = []
            for i in range(len(waves)):
                o = W.transcribe_clip(sd, cfg, sp, feats[i], language=lang)
                hf = net.generate(feats[i:i + 1].transpose(1, 2), **kw)
                hf_toks = hf[0].tolist()
                # generate's short-form output is the hypothesis without the prompt and without the eot it ended on
                mine = o["tokens"][:-1] if o["tokens"] and o["tokens"][-1] == sp["eot"] else o["tokens"]
                if mine != hf_toks:
                    raise AssertionError(f"{name} clip {i} lang {lang}: oracle {o['tokens']} != generate {hf_toks}")
                print(f"{name} clip {i} lang={lang} -> {o['language']}: {len(o['tokens'])} tokens identical to generate, "
                      f"score {o['score']:.4f}, no_speech {o['no_speech_prob']:.3e}")
                res.append(o)
            runs.append(dict(language=lang, results=res))
        out["cases"][name] = dict(cfg=cfg, seed=c["seed"], eot_gain=c["eot_gain"], secs=c["secs"], forced=toks,
                                  logits=lg.float(), runs=runs)
    torch.save(out, GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes")


if __name__ == "__main__":
    main()
