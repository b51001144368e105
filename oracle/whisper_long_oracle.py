"""Float64 restatement of long-form Whisper transcription as `whisper.WhisperModel.transcribe_long` runs it: transformers'
long-form `WhisperGenerationMixin.generate` (num_beams=5, return_timestamps=True, temperature=0.0,
condition_on_prev_tokens=False, logprob_threshold=-1.0, no_speech_threshold=0.6) for one clip of more than 3000 frames, on
the front end, network, processors and beam search of oracle/whisper_oracle.py.  oracle/pin_asr_long.py pins it against
transformers.
"""
import torch

from oracle.whisper_oracle import N_FRAMES, decode_logits, encode, log_mel, process, transcribe_clip

NO_SPEECH_THRESHOLD, LOGPROB_THRESHOLD = 0.6, -1.0


def window(lm, seek, n):
    """_get_input_segment: frames [seek, seek + n) of a whole-clip log_mel, zero after them -> [3000, n_mels]."""
    out = torch.zeros(N_FRAMES, lm.shape[1], dtype=torch.float64)
    out[:n] = lm[seek:seek + n]
    return out


def retrieve_segment(seq, ts_begin, n_frames):
    """_retrieve_segment: seq = the window's best hypothesis without its eot -> (tokens of its segments, seek offset in
    frames).  With consecutive timestamps and no single-timestamp ending, the segments end at the last pair and seek moves to
    the pair's first timestamp (input stride 2 frames per timestamp step); otherwise all tokens are kept and seek moves by
    the window."""
    ts = [t >= ts_begin for t in seq]
    single_ending = ts[-2:] == [False, True]
    idx = [i + 1 for i in range(len(seq) - 1) if ts[i] and ts[i + 1]]
    if idx and not single_ending:
        last = idx[-1] + 1
        return list(seq[:last]), 2 * (seq[last - 2] - ts_begin)
    return list(seq), n_frames


def avg_logprob(sd, cfg, sp, enc, prompt, tokens):
    """_retrieve_avg_logprobs of a hypothesis (its eot included): the mean over its tokens of log_softmax(processed
    log-probs)[token], the processed rows recomputed teacher-forced (a row depends only on its own prefix)."""
    lg = decode_logits(sd, enc, torch.tensor([list(prompt) + list(tokens[:-1])]), cfg)[0, len(prompt) - 1:]
    total = 0.0
    for t, tok in enumerate(tokens):
        lp = process(torch.log_softmax(lg[t:t + 1].float(), dim=-1), [list(tokens[:t])], sp)
        total += float(torch.log_softmax(lp, dim=-1)[0, tok])
    return total / len(tokens)


def transcribe_long(sd, cfg, sp, wave, language=None, num_beams=5, max_new_tokens=224):
    """The seek loop of one clip: the whole clip's log_mel, then 30 s windows from seek = 0 until seek >= its frames.  The
    language is detected on the first window when None and forced on the later ones; a window with no_speech_prob > 0.6
    and avg_logprob < -1.0 is skipped (no tokens, seek + its frames).  -> dict(language, tokens: the windows' kept tokens
    in order, windows: per window dict(seek, n_frames, tokens, kept, score, avg_logprob, no_speech_prob, skipped))."""
    lm = log_mel(wave, cfg["num_mel_bins"])
    frames, seek, windows, eot = lm.shape[0], 0, [], sp["eot"]
    while seek < frames:
        n = min(N_FRAMES, frames - seek)
        feats = window(lm, seek, n)
        o = transcribe_clip(sd, cfg, sp, feats, language, num_beams, max_new_tokens)
        language = o["language"]
        prompt = [sp["sot"], sp["langs"][language], sp["transcribe"]]
        alp = avg_logprob(sd, cfg, sp, encode(sd, feats[None], cfg), prompt, o["tokens"])
        seq = o["tokens"][:-1] if o["tokens"] and o["tokens"][-1] == eot else o["tokens"]
        skipped = o["no_speech_prob"] > NO_SPEECH_THRESHOLD and alp < LOGPROB_THRESHOLD
        kept, off = ([], n) if skipped else retrieve_segment(seq, sp["ts_begin"], n)
        windows.append(dict(seek=seek, n_frames=n, tokens=o["tokens"], kept=kept, score=o["score"], avg_logprob=alp,
                            no_speech_prob=o["no_speech_prob"], skipped=skipped))
        seek += off
    return dict(language=language, tokens=[t for w in windows for t in w["kept"]], windows=windows)
