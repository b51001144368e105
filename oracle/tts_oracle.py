"""Oracle of the synthesis call (easevoice-trainer_b200/tts.py): the numpy restatement of TTS.audio_postprocess
(reference src/easevoice/inference/tts.py:878-907) that evk_fragment_int16 is checked against, and the seeded inputs,
models and text front-end stand-in of the end-to-end cases that oracle/pin_tts.py runs through the reference's TTS.run and
tests/test_gpu_tts.py through tts.run (golden: tests/golden/tts.pt).
"""
import numpy as np
import torch

from oracle import gpt_oracle, hubert_oracle, s2_oracle
from oracle.slicer_oracle import to_int16

SR = 32000
GPT_SEED, S2_SEED, HUBERT_SEED, HUBERT_LAYERS = 14, 1234, 41, 2
HZ, MAX_SEC = 5, 2                       # early_stop_num = HZ * MAX_SEC = 10 tokens a sentence keeps the golden small
LANGS = ["auto", "auto_yue", "en", "zh", "ja", "yue", "ko", "all_zh", "all_ja", "all_yue", "all_ko"]   # TTSConfig.languages


def recovery_order(data, batch_index_list):
    out = [None] * len(sum(batch_index_list, []))
    for i, index_list in enumerate(batch_index_list):
        for j, index in enumerate(index_list):
            out[index] = data[i][j]
    return out


def audio_postprocess(audio, sr, batch_index_list=None, split_bucket=True, fragment_interval=0.3):
    """audio[i][j]: float32 samples of sentence j of bucket i -> (sr, int16): per fragment m = max |x| (NaN propagates),
    x / m when m > 1, int(sr * fragment_interval) zeros appended; sentence order (split_bucket) or bucket order; * 32768 and
    x86 numpy's astype(np.int16).  ValueError on an empty fragment (the reference's torch max raises RuntimeError)."""
    zero = np.zeros(int(sr * fragment_interval), dtype=np.float32)
    out = []
    for batch in audio:
        row = []
        for a in batch:
            a = np.asarray(a, dtype=np.float32)
            m = np.abs(a).max()
            if m > 1:
                a = a / m
            row.append(np.concatenate([a, zero]))
        out.append(row)
    flat = recovery_order(out, batch_index_list) if split_bucket else sum(out, [])
    return sr, to_int16(np.concatenate(flat) * np.float32(32768))


def synthetic_fragments():
    """-> [(name, audio, batch_index_list, split_bucket, fragment_interval)]: the edge cases of the conversion"""
    g = np.random.default_rng(5)

    def wave(n, peak=0.8):
        a = (np.tanh(g.standard_normal(n) * 2.0) * peak).astype(np.float32)
        return a

    one = wave(700, 0.9)
    one[123] = 1.0                                        # max exactly 1.0: not divided, 1.0 * 32768 wraps to -32768
    loud = wave(513, 1.2)
    loud[77] = 1.7                                        # unique peak above 1: divided, the peak becomes exactly 1.0
    neg = wave(640, 0.5)
    neg[5] = -1.5                                         # negative peak
    nan = wave(300)
    nan[17] = np.nan                                      # NaN max: no division, NaN converts to 0
    return [
        ("edges", [[one, loud], [neg, np.zeros(333, np.float32)], [nan]], [[3, 0], [1, 4], [2]], True, 0.3),
        ("bucket_order", [[wave(1000), wave(1)], [wave(77, 3.0)]], None, False, 0.01),
        ("empty", [[wave(50), np.zeros(0, np.float32)]], None, False, 0.3),
    ]


def bucket_cases(n=300, seed=11):
    """-> [(lengths, batch_size, threshold)]: random to_batch inputs"""
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(g.integers(1, 25))
        hi = int(g.choice([3, 10, 60]))
        out.append(([int(v) for v in g.integers(1, hi + 1, k)], int(g.integers(1, 9)), float(g.choice([0.0, 0.5, 0.75, 0.9, 1.0, 1.3]))))
    return out


# ---- end-to-end cases -------------------------------------------------------------------------------------------------------

CASES = {
    "prompt_buckets": dict(n_sent=7, inputs=dict(prompt_text="prompt", batch_size=3, split_bucket=True, speed_factor=1.0,
                                                 fragment_interval=0.05)),
    "ref_free_parallel": dict(n_sent=3, inputs=dict(prompt_text="", batch_size=2, parallel_infer=True, fragment_interval=0.3)),
    "ref_free_naive": dict(n_sent=3, inputs=dict(prompt_text="", batch_size=2, parallel_infer=False, fragment_interval=0.05)),
    "speed": dict(n_sent=3, inputs=dict(prompt_text="prompt", batch_size=3, speed_factor=1.25, fragment_interval=0.05)),
    "fragments": dict(n_sent=4, inputs=dict(prompt_text="prompt", batch_size=2, return_fragment=True, fragment_interval=0.05)),
    "aux_ref": dict(n_sent=2, inputs=dict(prompt_text="prompt", batch_size=2, aux_ref_audio_paths=["aux.wav"],
                                          fragment_interval=0.005)),
}
COMMON = dict(text="text", text_lang="zh", prompt_lang="zh", ref_audio_path="ref.wav", top_k=1, top_p=1, temperature=1,
              seed=1, repetition_penalty=1.35)


def case_inputs(name, paths):
    """the inputs dict of a case; paths maps the clip names to existing files"""
    d = dict(COMMON, **CASES[name]["inputs"])
    d["ref_audio_path"] = paths[d["ref_audio_path"]]
    d["aux_ref_audio_paths"] = [paths[p] for p in d.get("aux_ref_audio_paths", [])]
    return d


def sentences(n, seed):
    """n sentences of seeded phones, BERT features and norm_text (whose length sets the buckets)"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = int(torch.randint(6, 20, (1,), generator=g))
        out.append({"phones": torch.randint(0, 732, (x,), generator=g).tolist(), "bert_features": torch.randn(1024, x, generator=g),
                    "norm_text": "t" * int(torch.randint(2, 30, (1,), generator=g))})
    return out


def clips(seed):
    """{name: (samples at 32 kHz, samples at 16 kHz)} of the reference clip and the aux clip (3 s; the aux clip peaks above 1)"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, amp in (("ref.wav", 0.4), ("aux.wav", 1.6)):
        t = torch.arange(96000) / 32000.0
        f0 = 120 + 80 * torch.rand(1, generator=g)
        x32 = (amp * torch.sin(2 * np.pi * f0 * t) * (0.6 + 0.4 * torch.sin(2 * np.pi * 3 * t))
               + 0.05 * torch.randn(96000, generator=g)).float()
        out[name] = (x32.numpy(), x32[::2].contiguous().numpy())
    return out


class StubPreprocessor:
    """TextPreprocessor with fixed seeded results: preprocess -> the case's sentences, pre_seg_text -> their keys,
    segment_and_extract_feature_for_text -> a sentence by key, or the prompt's features for the prompt text"""

    def __init__(self, n_sent, seed):
        self.sent = sentences(n_sent, seed)
        self.prompt = sentences(1, seed + 1000)[0]

    def preprocess(self, text, lang, method):
        return [dict(s) for s in self.sent]

    def pre_seg_text(self, text, lang, method):
        return [f"s{i}" for i in range(len(self.sent))]

    def segment_and_extract_feature_for_text(self, text, lang):
        s = self.sent[int(text[1:])] if text.startswith("s") else self.prompt
        return list(s["phones"]), s["bert_features"].clone(), s["norm_text"]


def gpt_params():
    m = dict(gpt_oracle.GPT_MODEL, n_layer=3)
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), GPT_SEED)
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    return m, P


def s2_params():
    return dict(s2_oracle.S2_MODEL), s2_oracle.init_params(s2_oracle.generator_param_spec(), S2_SEED)


def hubert_params():
    m = dict(hubert_oracle.HUBERT_BASE, layers=HUBERT_LAYERS)
    return m, hubert_oracle.init_params(hubert_oracle.param_spec(m), HUBERT_SEED)


class NoiseStream:
    """the vocoder's normal draws, in call order: torch.randn of the requested shape from one seeded CPU generator"""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def draw(self, shape):
        return torch.randn(tuple(shape), generator=self.g)
