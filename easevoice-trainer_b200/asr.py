"""`WhisperAsr` (reference src/audiokit/asr/asr.py:68-148) on the library's Whisper (whisper.py): transcribe the clips that
`AudioService.slicer` writes into `asr.list` lines `file|lang|text`.

Differences from the reference, which runs faster-whisper: the model is a local Hugging Face Whisper directory (config.json,
model.safetensors or pytorch_model.bin, generation_config.json, tokenizer.json), decoding follows transformers' `generate`
(5 beams, timestamps, at most 224 new tokens per 30 s window) without the temperature-fallback ladder, conditioning on the
previous window or the VAD filter, and clips are decoded in batches.  `precision` "float16" and "bfloat16" run every Linear
on the library's 16-bit kernels (whisper.py); every other compute_type computes in fp32 with TF32 products.  Clips of at most 30 s are decoded whole; longer ones
follow transformers' long-form generate (30 s windows moved by the predicted timestamps, `WhisperModel.transcribe_long`),
with the windows of several clips decoded together.  See INTEGRATION.md.
"""
import os
import zlib

import numpy as np
import torch

from .utils.response import EaseVoiceResponse, ResponseStatus

VALID_SIZES = ["tiny", "tiny.en", "base", "base.en", "small", "small.en", "distil-small.en", "medium", "medium.en",
               "distil-medium.en", "large-v1", "large-v2", "large-v3", "large", "distil-large-v2", "distil-large-v3",
               "large-v3-turbo", "turbo"]
VALID_LANGUAGES = [
    "af", "am", "ar", "as", "az", "ba", "be", "bg", "bn", "bo", "br", "bs", "ca", "cs", "cy", "da", "de", "el", "en", "es",
    "et", "eu", "fa", "fi", "fo", "fr", "gl", "gu", "ha", "haw", "he", "hi", "hr", "ht", "hu", "hy", "id", "is", "it", "ja",
    "jw", "ka", "kk", "km", "kn", "ko", "la", "lb", "ln", "lo", "lt", "lv", "mg", "mi", "mk", "ml", "mn", "mr", "ms", "mt",
    "my", "ne", "nl", "nn", "no", "oc", "pa", "pl", "ps", "pt", "ro", "ru", "sa", "sd", "si", "sk", "sl", "sn", "so", "sq",
    "sr", "su", "sv", "sw", "ta", "te", "tg", "th", "tk", "tl", "tr", "tt", "uk", "ur", "uz", "vi", "yi", "yo", "zh", "yue",
    "auto"]
# faster-whisper's defaults: a clip whose first pass puts more than 0.6 on <|nospeech|> and whose best hypothesis averages
# below -1.0 log-prob per token has no text
NO_SPEECH_THRESHOLD, LOGPROB_THRESHOLD = 0.6, -1.0
# device memory for one batch's per-clip buffers: cross K/V (1500 x layers x 2 d fp32) and the self-attention slots of its
# 5 beams (448 x layers x 2 d fp32 each).  large-v3: 0.49 GB + 0.73 GB per clip, so 16 GiB holds 14 clips
DEFAULT_MEMORY_BUDGET = 16 << 30
# share of the budget for a pool of long clips' whole-clip log-mels (fp32 [frames, n_mels]; large-v3: 512 bytes per 10 ms, so
# 2 GiB of a 16 GiB budget holds about 11.6 hours of audio); the decode batch of long clips takes the rest
LONG_POOL_SHARE = 1 / 8
# faster-whisper compute_type values that select the 16-bit Linears.  The others ("float32", "int8*", "default", "auto")
# are accepted and recorded, and compute in fp32 with TF32 products.
H16_PRECISIONS = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def compute_dtype(precision):
    """WhisperModel compute type of a compute_type value: torch.float16 / torch.bfloat16, or None (fp32 / TF32)."""
    return H16_PRECISIONS.get(precision)


def read_clip(path, max_seconds=30):
    """-> float32 16 kHz samples of a 16 or 32 kHz wav (32 kHz through resample_poly(x, 1, 2) with the SSL taps), or raises
    ValueError.  int16 is scaled by 1 / 32768, float is taken as it is; other sample formats are rejected.  max_seconds: the
    longest clip accepted (None: any length)."""
    from scipy.io import wavfile
    sr, x = wavfile.read(path)
    if sr not in (16000, 32000):
        raise ValueError(f"{path}: sample rate {sr} (16 or 32 kHz)")
    if x.ndim != 1:
        raise ValueError(f"{path}: {x.ndim}-D audio (mono only)")
    if x.dtype == np.int16:
        x = x.astype(np.float32) / 32768.0
    elif x.dtype in (np.float32, np.float64):
        x = x.astype(np.float32)
    else:
        raise ValueError(f"{path}: {x.dtype} samples (int16 or float)")
    n16 = x.size if sr == 16000 else (x.size + 1) // 2
    if max_seconds is not None and n16 > max_seconds * 16000:
        raise ValueError(f"{path}: {n16 / 16000:.2f} s (clips of at most {max_seconds} s)")
    if n16 < 201:
        raise ValueError(f"{path}: {n16} samples at 16 kHz (at least 201)")
    return x, sr


def decode_text(tokenizer, tokens, eot):
    """Text of a hypothesis: its text tokens (ids below eot) decoded and joined; timestamps and special tokens dropped."""
    return tokenizer.decode([t for t in tokens if t < eot])


def compression_ratio(text):
    b = text.encode("utf-8")
    return len(b) / len(zlib.compress(b)) if b else 0.0


def is_no_speech(no_speech_prob, avg_logprob):
    return no_speech_prob > NO_SPEECH_THRESHOLD and avg_logprob < LOGPROB_THRESHOLD


def clips_per_batch(cfg, budget=DEFAULT_MEMORY_BUDGET, beams=5):
    per = 4 * cfg["decoder_layers"] * 2 * cfg["d_model"] * (1500 + beams * cfg["max_target_positions"])
    return max(1, int(budget // per))


def samples_16k(x, sr):
    return x.size if sr == 16000 else (x.size + 1) // 2


def long_pools(n16, n_mels, budget=DEFAULT_MEMORY_BUDGET):
    """Consecutive groups of the long clips (16 kHz sample counts n16, in list order) whose whole-clip log-mel buffer
    [clips, longest // 160, n_mels] fp32 fits LONG_POOL_SHARE of the budget; a clip too long for it alone is a pool of one.
    -> list of lists of indices into n16."""
    cap, pools = budget * LONG_POOL_SHARE, []
    for i, n in enumerate(n16):
        if pools:
            p = pools[-1]
            T = max(n, max(n16[j] for j in p)) // 160
            if (len(p) + 1) * T * n_mels * 4 <= cap:
                p.append(i)
                continue
        pools.append([i])
    return pools


class WhisperAsr:
    def __init__(self, model_size: str, language: str, precision: str, model_dir=None, memory_budget=DEFAULT_MEMORY_BUDGET):
        """model_size and language are validated as the reference does.  precision takes the reference's compute_type values:
        "float16" and "bfloat16" run the Linears on the 16-bit kernels (compute_dtype); the others are recorded and compute
        in fp32 with TF32 tensor-core products.  Cross K/V and the decode slots stay fp32 either way, so the batch size
        (clips_per_batch) is the same.  model_dir: the local Hugging Face Whisper directory (default: the directory named
        model_size)."""
        if model_size not in VALID_SIZES:
            raise ValueError(f"Invalid model size: {model_size}")
        if language not in VALID_LANGUAGES:
            raise ValueError(f"Invalid language: {language}")
        self.model_path = model_dir or model_size
        self.language = language if language != "auto" else None
        self.precision = precision
        self.memory_budget = memory_budget

    def load(self):
        """-> (WhisperModel on cuda, tokenizers.Tokenizer of the model directory's tokenizer.json), loaded on the first call
        and kept, so later calls reuse the model and its captured decode graph."""
        if getattr(self, "_loaded", None) is None:
            from tokenizers import Tokenizer

            from .whisper import WhisperModel
            self._loaded = (WhisperModel.from_pretrained(self.model_path, device="cuda", compute_type=compute_dtype(self.precision)),
                            Tokenizer.from_file(os.path.join(self.model_path, "tokenizer.json")))
        return self._loaded

    def recognize(self, file_list: list, output_file: str, dump_file: str) -> EaseVoiceResponse:
        from . import ops
        from .normalize_ssl import resample_taps
        try:
            model, tokenizer = self.load()
        except Exception as e:       # noqa: BLE001  (the reference reports any load failure this way)
            print(f"Failed to load model: {e!r}")
            return EaseVoiceResponse(status=ResponseStatus.FAILED, message="Failed to load model")
        if self.language is not None and self.language not in model.sp["langs"]:
            print(f"language {self.language!r} is not in the model's generation config")
            return EaseVoiceResponse(status=ResponseStatus.FAILED, message=f"Language {self.language} is not supported by the model")
        trace_data, clips = {}, []
        for f in file_list:                                  # validate every file first, in list order
            try:
                clips.append(read_clip(f, max_seconds=None))
            except Exception as e:   # noqa: BLE001
                print(f"{f}: {e!r}")
                trace_data[f] = ResponseStatus.FAILED
                return EaseVoiceResponse(status=ResponseStatus.FAILED, message="Failed to recognize audio", data=trace_data)
            trace_data[f] = ResponseStatus.SUCCESS
        dev = torch.device("cuda", torch.cuda.current_device())
        h = torch.from_numpy(resample_taps()[1]).to(dev)
        nb, sp, lines, info = clips_per_batch(model.cfg, self.memory_budget), model.sp, {}, {}

        def wav_rows(idx):
            rows = []
            for i in idx:
                x, sr = clips[i]
                xd = torch.from_numpy(x).to(dev)[None]
                if sr == 32000:
                    xd = ops.resample_poly(xd, h, 1, 2, 64, (x.size + 1) // 2)
                rows.append(xd[0])
            wav = torch.zeros(len(rows), max(r.numel() for r in rows), device=dev)
            for i, r in enumerate(rows):
                wav[i, :r.numel()] = r
            return wav, [r.numel() for r in rows]

        n16 = [samples_16k(x, sr) for x, sr in clips]
        short = [i for i, n in enumerate(n16) if n <= 30 * 16000]
        long = [i for i, n in enumerate(n16) if n > 30 * 16000]
        for s in range(0, len(short), nb):                  # clips of at most 30 s: whole, in batches of nb
            idx = short[s:s + nb]
            feats = model.features(*wav_rows(idx))
            for i, o in zip(idx, model.transcribe_features(feats, language=self.language)):
                f = file_list[i]
                text = decode_text(tokenizer, o["tokens"], sp["eot"])
                if is_no_speech(o["no_speech_prob"], o["score"]):
                    text = ""
                lines[i] = f"{f}|{o['language'].lower()}|{text}"
                info[f] = dict(status=ResponseStatus.SUCCESS, avg_logprob=o["score"], compression_ratio=compression_ratio(text),
                               no_speech_prob=o["no_speech_prob"])
        nb_long = clips_per_batch(model.cfg, self.memory_budget * (1 - LONG_POOL_SHARE))
        for pool in long_pools([n16[i] for i in long], model.cfg["num_mel_bins"], self.memory_budget):
            idx = [long[j] for j in pool]                    # longer clips: 30 s windows, pool by pool
            wav, lens = wav_rows(idx)
            lm = model.features_long(wav, lens)
            del wav
            res = model.transcribe_long(lm, [n // 160 for n in lens], language=self.language, clips_per_batch=nb_long)
            del lm
            for i, o in zip(idx, res):
                f, ws = file_list[i], o["windows"]
                text = decode_text(tokenizer, o["tokens"], sp["eot"])
                lines[i] = f"{f}|{o['language'].lower()}|{text}"
                spoken = [w["avg_logprob"] for w in ws if not w["skipped"]] or [ws[0]["avg_logprob"]]
                info[f] = dict(status=ResponseStatus.SUCCESS, avg_logprob=sum(spoken) / len(spoken),
                               compression_ratio=compression_ratio(text), no_speech_prob=ws[0]["no_speech_prob"],
                               windows=[dict(start_s=w["seek"] / 100, end_s=(w["seek"] + w["n_frames"]) / 100,
                                             avg_logprob=w["avg_logprob"], no_speech_prob=w["no_speech_prob"],
                                             skipped=w["skipped"]) for w in ws])
        output, info = [lines[i] for i in range(len(file_list))], {f: info[f] for f in file_list}
        with open(output_file, "w", encoding="utf-8") as fo:
            fo.write("\n".join(output))
        with open(dump_file, "w", encoding="utf-8") as fo:
            fo.write("\n".join(output))
        return EaseVoiceResponse(status=ResponseStatus.SUCCESS, message="asr success", data=info)
