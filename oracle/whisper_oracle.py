"""Float64 restatement of Whisper transcription as `whisper.py` runs it: the log-mel front end, the encoder and decoder of
transformers' `WhisperForConditionalGeneration`, the logits processors of its `generate(return_timestamps=True)` and the
beam search of `GenerationMixin._beam_search`.  oracle/pin_asr.py pins every piece against transformers.

Beam bookkeeping is float32, as in transformers: `_beam_search` casts the logits to float32 before `log_softmax`.
"""
import math

import numpy as np
import torch

N_FFT, HOP, SR, N_FRAMES, N_AUDIO_CTX = 400, 160, 16000, 3000, 1500
NEG = -1.0e9


# ---- front end ------------------------------------------------------------------------------------------------------------
def mel_filters(n_mels):
    """transformers' mel_filter_bank(201, n_mels, 0, 8000, 16000, norm="slaney", mel_scale="slaney") -> [201, n_mels]."""
    def hz2mel(f):
        f = np.asarray(f, dtype=np.float64)
        m = 3.0 * f / 200.0
        return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-12) / 1000.0) * (27.0 / np.log(6.4)), m)

    def mel2hz(m):
        m = np.asarray(m, dtype=np.float64)
        f = 200.0 * m / 3.0
        return np.where(m >= 15.0, 1000.0 * np.exp(np.log(6.4) / 27.0 * (m - 15.0)), f)

    ff = mel2hz(np.linspace(hz2mel(0.0), hz2mel(8000.0), n_mels + 2))
    fft = np.linspace(0, SR // 2, N_FFT // 2 + 1)
    slopes = ff[None, :] - fft[:, None]
    d = np.diff(ff)
    fb = np.maximum(0.0, np.minimum(-slopes[:, :-2] / d[:-1], slopes[:, 2:] / d[1:]))
    return fb * (2.0 / (ff[2:] - ff[:-2]))[None, :]


def num_frames(n_samples):
    """Frames of a clip of n 16 kHz samples: the centred STFT has 1 + n // 160, the last of which every Whisper front end drops."""
    return int(n_samples) // HOP


def log_mel(wave, n_mels):
    """wave: 1-D 16 kHz samples -> [num_frames(n), n_mels] float64, normalised over the clip's own frames."""
    x = torch.as_tensor(np.asarray(wave, dtype=np.float64))
    T = num_frames(x.numel())
    xp = torch.nn.functional.pad(x[None, None], (N_FFT // 2, N_FFT // 2), mode="reflect")[0, 0]
    fr = xp.unfold(0, N_FFT, HOP)[:T]
    n = torch.arange(N_FFT, dtype=torch.float64)
    win = 0.5 - 0.5 * torch.cos(2 * math.pi * n / N_FFT)                      # periodic Hann
    spec = torch.fft.rfft(fr * win, dim=-1).abs() ** 2
    mel = spec @ torch.as_tensor(mel_filters(n_mels))
    lm = torch.log10(torch.clamp(mel, min=1e-10))
    lm = torch.maximum(lm, lm.max() - 8.0)
    return (lm + 4.0) / 4.0


def features(wave, n_mels):
    """[3000, n_mels]: log_mel of the clip, zero after its frames (padding in the feature domain, openai-whisper's
    pad_or_trim of the normalised log-mel).  A clip over 30 s has more than 3000 frames and raises."""
    lm = log_mel(wave, n_mels)
    if lm.shape[0] > N_FRAMES:
        raise ValueError("clip longer than 30 s")
    out = torch.zeros(N_FRAMES, n_mels, dtype=torch.float64)
    out[:lm.shape[0]] = lm
    return out


# ---- network ---------------------------------------------------------------------------------------------------------------
def param_spec(cfg):
    """(name, shape) of WhisperForConditionalGeneration's state_dict without the tied proj_out.weight."""
    d, M, V = cfg["d_model"], cfg["num_mel_bins"], cfg["vocab_size"]
    out = [("model.encoder.conv1.weight", (d, M, 3)), ("model.encoder.conv1.bias", (d,)),
           ("model.encoder.conv2.weight", (d, d, 3)), ("model.encoder.conv2.bias", (d,)),
           ("model.encoder.embed_positions.weight", (cfg["max_source_positions"], d))]

    def attn(p):
        r = []
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            r.append((p + n + ".weight", (d, d)))
            if n != "k_proj":
                r.append((p + n + ".bias", (d,)))
        return r

    def block(p, ffn, cross):
        r = attn(p + "self_attn.") + [(p + "self_attn_layer_norm.weight", (d,)), (p + "self_attn_layer_norm.bias", (d,))]
        if cross:
            r += attn(p + "encoder_attn.") + [(p + "encoder_attn_layer_norm.weight", (d,)),
                                              (p + "encoder_attn_layer_norm.bias", (d,))]
        return r + [(p + "fc1.weight", (ffn, d)), (p + "fc1.bias", (ffn,)), (p + "fc2.weight", (d, ffn)), (p + "fc2.bias", (d,)),
                    (p + "final_layer_norm.weight", (d,)), (p + "final_layer_norm.bias", (d,))]

    for i in range(cfg["encoder_layers"]):
        out += block(f"model.encoder.layers.{i}.", cfg["encoder_ffn_dim"], False)
    out += [("model.encoder.layer_norm.weight", (d,)), ("model.encoder.layer_norm.bias", (d,)),
            ("model.decoder.embed_tokens.weight", (V, d)), ("model.decoder.embed_positions.weight", (cfg["max_target_positions"], d))]
    for i in range(cfg["decoder_layers"]):
        out += block(f"model.decoder.layers.{i}.", cfg["decoder_ffn_dim"], True)
    return out + [("model.decoder.layer_norm.weight", (d,)), ("model.decoder.layer_norm.bias", (d,))]


def _ln(x, sd, p, eps=1e-5):
    return torch.nn.functional.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], eps)


def _lin(x, sd, p, bias=True):
    y = x @ sd[p + ".weight"].T
    return y + sd[p + ".bias"] if bias else y


def _mha(x, kv, sd, p, H, causal):
    B, T, D = x.shape
    q = _lin(x, sd, p + ".q_proj").view(B, T, H, -1).transpose(1, 2)
    k = _lin(kv, sd, p + ".k_proj", bias=False).view(B, kv.shape[1], H, -1).transpose(1, 2)
    v = _lin(kv, sd, p + ".v_proj").view(B, kv.shape[1], H, -1).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * (D // H) ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool).triu(1), float("-inf"))
    a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, T, D)
    return _lin(a, sd, p + ".out_proj")


def _gelu(x):
    return torch.nn.functional.gelu(x)


def encode(sd, feats, cfg):
    """feats [B, 3000, n_mels] -> encoder last_hidden_state [B, 1500, d_model] (float64)."""
    sd = {k: v.double() for k, v in sd.items()}
    x = feats.double().transpose(1, 2)
    x = _gelu(torch.nn.functional.conv1d(x, sd["model.encoder.conv1.weight"], sd["model.encoder.conv1.bias"], padding=1))
    x = _gelu(torch.nn.functional.conv1d(x, sd["model.encoder.conv2.weight"], sd["model.encoder.conv2.bias"], stride=2, padding=1))
    h = x.transpose(1, 2) + sd["model.encoder.embed_positions.weight"]
    H = cfg["encoder_attention_heads"]
    for i in range(cfg["encoder_layers"]):
        p = f"model.encoder.layers.{i}."
        h = h + _mha(_ln(h, sd, p + "self_attn_layer_norm"), _ln(h, sd, p + "self_attn_layer_norm"), sd, p + "self_attn", H, False)
        h = h + _lin(_gelu(_lin(_ln(h, sd, p + "final_layer_norm"), sd, p + "fc1")), sd, p + "fc2")
    return _ln(h, sd, "model.encoder.layer_norm")


def decode_logits(sd, enc, tokens, cfg):
    """Teacher-forced decoder: enc [B, 1500, d], tokens [B, T] int64 -> logits [B, T, V] (float64)."""
    sd = {k: v.double() for k, v in sd.items()}
    T = tokens.shape[1]
    h = sd["model.decoder.embed_tokens.weight"][tokens] + sd["model.decoder.embed_positions.weight"][:T]
    H = cfg["decoder_attention_heads"]
    enc = enc.double()
    for i in range(cfg["decoder_layers"]):
        p = f"model.decoder.layers.{i}."
        a = _ln(h, sd, p + "self_attn_layer_norm")
        h = h + _mha(a, a, sd, p + "self_attn", H, True)
        h = h + _mha(_ln(h, sd, p + "encoder_attn_layer_norm"), enc, sd, p + "encoder_attn", H, False)
        h = h + _lin(_gelu(_lin(_ln(h, sd, p + "final_layer_norm"), sd, p + "fc1")), sd, p + "fc2")
    h = _ln(h, sd, "model.decoder.layer_norm")
    return h @ sd["model.decoder.embed_tokens.weight"].T


# ---- special tokens and logits processors ---------------------------------------------------------------------------------
def special_tokens(gen):
    """Ids that decoding needs, from a generation_config.json mapping."""
    nots = int(gen["no_timestamps_token_id"])
    return dict(sot=int(gen["decoder_start_token_id"]), eot=int(gen["eos_token_id"]), notimestamps=nots, ts_begin=nots + 1,
                nospeech=nots - 1, transcribe=int(gen["task_to_id"]["transcribe"]),
                langs={k[2:-2]: int(v) for k, v in gen["lang_to_id"].items()},
                suppress=[int(t) for t in gen.get("suppress_tokens") or []],
                begin_suppress=[int(t) for t in gen.get("begin_suppress_tokens") or []],
                max_initial_ts=gen.get("max_initial_timestamp_index"))


def process(lp, gen_seqs, sp):
    """transformers' processors on log-probs (float32 [R, V]) in generate's order: SuppressTokensAtBegin, SuppressTokens,
    WhisperTimeStamp.  gen_seqs: per row, the tokens generated after the prompt."""
    lp = lp.clone()
    V = lp.shape[1]
    tb, eot = sp["ts_begin"], sp["eot"]
    first = len(gen_seqs[0]) == 0
    if first and sp["begin_suppress"]:
        lp[:, [t for t in sp["begin_suppress"] if t < V]] = float("-inf")
    if sp["suppress"]:
        lp[:, [t for t in sp["suppress"] if t < V]] = float("-inf")
    lp[:, sp["notimestamps"]] = float("-inf")
    for k, seq in enumerate(gen_seqs):
        last_ts = len(seq) >= 1 and seq[-1] >= tb
        pen_ts = len(seq) < 2 or seq[-2] >= tb
        if last_ts:
            if pen_ts:
                lp[k, tb:] = float("-inf")
            else:
                lp[k, :eot] = float("-inf")
        ts = [t for t in seq if t >= tb]
        if ts:
            lim = ts[-1] if (last_ts and not pen_ts) else ts[-1] + 1
            lp[k, tb:lim] = float("-inf")
    if first:
        lp[:, :tb] = float("-inf")
        if sp["max_initial_ts"] is not None:
            lp[:, tb + int(sp["max_initial_ts"]) + 1:] = float("-inf")
    l2 = torch.log_softmax(lp.float(), dim=-1)
    for k in range(lp.shape[0]):
        if l2[k, tb:].logsumexp(-1) > l2[k, :tb].max():
            lp[k, :tb] = float("-inf")
    return lp


# ---- beam search ------------------------------------------------------------------------------------------------------------
def beam_step(lp, run, run_sc, fin, fin_sc, fin_done, unsat, plen, max_length, eot, length_penalty=1.0):
    """One iteration of `_beam_search` (early_stopping=False) for one clip.  lp: processed log-probs float32 [beams, V];
    run: the beams' token lists (prompt included); run_sc float32 [beams]; fin / fin_sc / fin_done: the finished set; unsat:
    the early-stop flag.  -> dict(run, run_sc, parent, tok, fin, fin_sc, fin_done, unsat, all_hit)."""
    num_beams, V = lp.shape
    K = 2 * num_beams
    cur = len(run[0])
    acc = (lp + run_sc[:, None]).reshape(-1)
    tv, ti = torch.topk(acc, K)
    par, tok = (ti // V).tolist(), (ti % V).tolist()
    cand = [run[p] + [t] for p, t in zip(par, tok)]
    hits = torch.tensor([t == eot or cur + 1 >= max_length for t in tok])
    rv = tv + hits.float() * NEG
    nxt = torch.topk(rv, num_beams)[1].tolist()
    did = hits & (torch.arange(K) < num_beams)
    fs = tv / ((cur + 1 - plen) ** length_penalty)
    fs = fs + (0.0 if unsat else 1.0) * NEG
    fs = fs + (~did).float() * NEG
    msc = torch.cat([fin_sc, fs])
    mseq = list(fin) + cand
    mdone = list(fin_done) + did.tolist()
    top = torch.topk(msc, num_beams)[1].tolist()
    fin, fin_sc, fin_done = [mseq[i] for i in top], msc[top], [mdone[i] for i in top]
    run_sc = rv[nxt]
    best_run = run_sc[0] / ((cur + 1 - plen) ** length_penalty)
    worst = torch.where(torch.tensor(fin_done), fin_sc.min(), torch.tensor(NEG))
    unsat = unsat and bool((best_run > worst).any())
    return dict(run=[cand[i] for i in nxt], run_sc=run_sc, parent=[par[i] for i in nxt], tok=[tok[i] for i in nxt], fin=fin,
                fin_sc=fin_sc, fin_done=fin_done, unsat=unsat, all_hit=bool(hits.all()))


def beam_search(logits_fn, prompt, sp, num_beams=5, max_new_tokens=224, length_penalty=1.0):
    """`_beam_search` for one clip, early_stopping=False.  logits_fn(list of token lists) -> float64/32 logits [rows, V] of
    the last position.  -> (generated tokens of the best hypothesis incl. eot, its length-normalised score)."""
    plen = len(prompt)
    run = [list(prompt) for _ in range(num_beams)]
    run_sc = torch.full((num_beams,), NEG, dtype=torch.float32)
    run_sc[0] = 0.0
    fin = [list(prompt) for _ in range(num_beams)]
    fin_sc = torch.full((num_beams,), NEG, dtype=torch.float32)
    fin_done = [False] * num_beams
    unsat = True
    while True:
        lp = process(torch.log_softmax(logits_fn(run).float(), dim=-1), [r[plen:] for r in run], sp)
        o = beam_step(lp, run, run_sc, fin, fin_sc, fin_done, unsat, plen, plen + max_new_tokens, sp["eot"], length_penalty)
        run, run_sc, fin, fin_sc, fin_done, unsat = o["run"], o["run_sc"], o["fin"], o["fin_sc"], o["fin_done"], o["unsat"]
        if not unsat or o["all_hit"]:
            break
    return fin[0][plen:], float(fin_sc[0])


def transcribe_clip(sd, cfg, sp, feats, language=None, num_beams=5, max_new_tokens=224):
    """One clip end to end: language detection when language is None, the no-speech probability at <|startoftranscript|>,
    beam search.  -> dict(language, tokens, score, no_speech_prob)."""
    enc = encode(sd, feats[None], cfg)
    l0 = decode_logits(sd, enc, torch.tensor([[sp["sot"]]]), cfg)[0, -1]
    langs = sp["langs"]
    lang_ids = torch.tensor(sorted(langs.values()))
    if language is None:
        lid = int(lang_ids[l0[lang_ids].argmax()])
        language = {v: k for k, v in langs.items()}[lid]
    nsp = float(torch.softmax(l0, -1)[sp["nospeech"]])
    prompt = [sp["sot"], langs[language], sp["transcribe"]]

    def fn(rows):
        return decode_logits(sd, enc.expand(len(rows), -1, -1), torch.tensor(rows), cfg)[:, -1]

    toks, score = beam_search(fn, prompt, sp, num_beams, max_new_tokens)
    return dict(language=language, tokens=toks, score=score, no_speech_prob=nsp)
