"""Voice-clone synthesis: the computing parts of the reference's `TTS` class (src/easevoice/inference/tts.py) on this library.

The caller keeps its `TTS` object, its `TextPreprocessor` (G2P stays on the host) and its file decoding (`load_audio`,
`librosa.load`); its models are this library's `models.SynthesizerTrn`, `models_gpt.Text2SemanticDecoder`,
`hubert.CNHubert` and `bert.BertModel` (INTEGRATION §3).  Each function here replaces one method body:

  ref_spec          `_get_ref_spec` after `load_audio`: the reference clip's linear spectrogram on the device
  prompt_semantic   `_set_prompt_semantic` after `librosa.load`: HuBERT features and semantic tokens of the reference clip
  to_batch          `to_batch`: sentences grouped into buckets of similar text length, tensors on the device
  recovery_order    `recovery_order`
  run               `run`: the whole synthesis generator
  run_many          several `run` requests in one call, their sentences decoded together (Text2SemanticDecoder.decode_groups)
  enable_half_precision  `enable_half_precision`: AR decoding in 16 bits (or back to fp32); the other models stay fp32
  audio_postprocess `audio_postprocess`: every fragment normalised, placed in sentence order, followed by its silent interval
                    and converted to int16 by one kernel (evk_fragment_int16); the int16 array crosses to the host once

The audio is the reference's, quirks included:
  * the prompt clip is padded with int(sampling_rate * 0.3) zeros although it is at 16 kHz: 0.6 s, not 0.3 s;
  * at speed_factor 1 every bucket is vocoded as one sequence (codes and phones of its sentences concatenated, so the
    attention of the prior encoder sees across sentence boundaries) and cut at 2 * prod(upsample_rates) samples per token;
    at any other speed each sentence is vocoded alone;
  * a sample of exactly 1.0 (tanh saturates to it) becomes 32768, which int16 wraps to -32768.
The sampling noise of `infer_panel` and `decode` is this library's device stream, not torch's CPU/CUDA generator: a seed
reproduces a run, but sampled tokens and the vocoder noise differ from the reference's (greedy decoding does not).
"""
import math
import os
import random

import numpy as np
import torch

from . import lib, ops
from .mel_processing import spectrogram_torch

SPLITS = {"，", "。", "？", "！", ",", ".", "?", "!", "~", ":", "：", "—", "…"}     # segmentation.py:9
PROMPT_MIN, PROMPT_MAX = 48000, 160000                                       # 3 to 10 s at 16 kHz


def set_seed(seed):
    """tts.py:35-51"""
    seed = int(seed)
    seed = seed if seed != -1 else random.randrange(1 << 32)
    os.environ["PYTHONHASHSEED"] = str(seed)
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
    return seed


def enable_half_precision(tts, enable=True, save=True):
    """`enable_half_precision` (tts.py:317-349) for what this library runs: the stage-1 GPT's AR decoding switches to 16-bit
    Linears and a 16-bit K/V cache (Text2SemanticDecoder.set_compute_type(torch.float16)), or back to fp32.  The vocoder, BERT
    and HuBERT stay in fp32 and are not touched.  On a CPU device, enabling does nothing (the reference logs and returns)."""
    if str(tts.configs.device) == "cpu" and enable:
        return
    tts.configs.is_half = enable
    tts.precision = torch.float16 if enable else torch.float32
    if save:
        tts.configs.save_configs()
    tts.t2s_model.model.set_compute_type(torch.float16 if enable else None)


def ref_spec(audio32k, filter_length, sampling_rate, hop_length, win_length, device):
    """`_get_ref_spec` (tts.py:390-409) after `load_audio`: audio32k 1-D float samples -> [1, filter_length // 2 + 1, T] fp32
    on device.  A clip whose max |x| exceeds 1 is divided by min(2, max |x|)."""
    x = torch.as_tensor(np.asarray(audio32k, dtype=np.float32)).to(device)
    m = x.abs().max()
    x = torch.where(m > 1, x / torch.clamp(m, max=2.0), x)
    return spectrogram_torch(x.unsqueeze(0), filter_length, sampling_rate, hop_length, win_length, center=False)


def prompt_semantic(wav16k, hubert_model, vits_model, sampling_rate):
    """`_set_prompt_semantic` (tts.py:411-437) after `librosa.load`: wav16k 1-D float samples at 16 kHz -> the int64 semantic
    tokens of the clip (1-D, on the models' device).  OSError for fewer than 3 s or more than 10 s, before any GPU work."""
    wav = np.asarray(wav16k, dtype=np.float32)
    if wav.ndim != 1:
        raise ValueError(f"prompt_semantic: expected mono samples, got shape {wav.shape}")
    if wav.shape[0] > PROMPT_MAX or wav.shape[0] < PROMPT_MIN:
        raise OSError("audio length should be in 3~10 seconds.")
    dev = next(hubert_model.model.parameters()).device
    x = torch.cat([torch.from_numpy(wav), torch.zeros(int(sampling_rate * 0.3))]).to(dev)
    with torch.no_grad():
        feat = hubert_model.model(x.unsqueeze(0))["last_hidden_state"].transpose(1, 2)
        codes = vits_model.extract_latent(feat)
    return codes[0, 0]


def to_batch(data, prompt_data=None, batch_size=5, threshold=0.75, split_bucket=True, device=torch.device("cpu")):
    """tts.py:460-551 -> (batches, batch_index_list).  With split_bucket, sentences sorted by len(norm_text) are cut into
    buckets of at most batch_size: a bucket is shortened from its end until its middle length over its mean length (float32)
    reaches threshold or it holds one sentence.  Without, consecutive groups of batch_size.  Tensors are fp32 / int64 on
    device."""
    index_and_len_list = [[idx, len(item["norm_text"])] for idx, item in enumerate(data)]
    batch_index_list = []
    if split_bucket:
        index_and_len_list.sort(key=lambda x: x[1])
        index_and_len_list = np.array(index_and_len_list, dtype=np.int64)
        pos = 0
        while pos < index_and_len_list.shape[0]:
            pos_end = min(pos + batch_size, index_and_len_list.shape[0])
            while pos < pos_end:
                batch = index_and_len_list[pos:pos_end, 1].astype(np.float32)
                score = batch[(pos_end - pos) // 2] / (batch.mean() + 1e-8)
                if (score >= threshold) or (pos_end - pos == 1):
                    batch_index_list.append(index_and_len_list[pos:pos_end, 0].tolist())
                    pos = pos_end
                    break
                pos_end = pos_end - 1
        assert sum(len(b) for b in batch_index_list) == len(data)
    else:
        for i in range(len(data)):
            if i % batch_size == 0:
                batch_index_list.append([])
            batch_index_list[-1].append(i)

    out = []
    for index_list in batch_index_list:
        phones_list, phones_len, all_phones_list, all_phones_len, all_bert, norm_text = [], [], [], [], [], []
        bert_max, phones_max = 0, 0
        for idx in index_list:
            item = data[idx]
            phones = torch.tensor(item["phones"], dtype=torch.int64, device=device)
            if prompt_data is not None:
                bert = torch.cat([prompt_data["bert_features"], item["bert_features"]], 1).to(dtype=torch.float32, device=device)
                all_phones = torch.tensor(prompt_data["phones"] + item["phones"], dtype=torch.int64, device=device)
            else:
                bert = item["bert_features"].to(dtype=torch.float32, device=device)
                all_phones = phones
            bert_max = max(bert_max, bert.shape[-1])
            phones_max = max(phones_max, all_phones.shape[-1])
            phones_list.append(phones)
            phones_len.append(phones.shape[-1])
            all_phones_list.append(all_phones)
            all_phones_len.append(all_phones.shape[-1])
            all_bert.append(bert)
            norm_text.append(item["norm_text"])
        out.append({
            "phones": phones_list,
            "phones_len": torch.tensor(phones_len, dtype=torch.int64, device=device),
            "all_phones": all_phones_list,
            "all_phones_len": torch.tensor(all_phones_len, dtype=torch.int64, device=device),
            "all_bert_features": all_bert,
            "norm_text": norm_text,
            "max_len": max(bert_max, phones_max),
        })
    return out, batch_index_list


def recovery_order(data, batch_index_list):
    """tts.py:553-569: data[i][j] is sentence batch_index_list[i][j] -> the list in sentence order"""
    _data = [None] * len(sum(batch_index_list, []))
    for i, index_list in enumerate(batch_index_list):
        for j, index in enumerate(index_list):
            _data[index] = data[i][j]
    return _data


def audio_postprocess(audio, sr, batch_index_list=None, speed_factor=1.0, split_bucket=True, fragment_interval=0.3):
    """tts.py:878-907: audio[i][j] the 1-D device waveform of sentence j of bucket i -> (sr, int16 ndarray): every fragment
    divided by its max |x| when that exceeds 1, followed by int(sr * fragment_interval) zeros, in sentence order
    (recovery_order) with split_bucket, in bucket order without, times 32768 and converted to int16 as x86 numpy's astype
    does.  One kernel writes the whole array on the device and it is copied to the host once."""
    order = [(i, j) for i, batch in enumerate(audio) for j in range(len(batch))]
    if split_bucket:
        order = recovery_order([[(i, j) for j in range(len(b))] for i, b in enumerate(audio)], batch_index_list)
    if not order:
        raise ValueError("need at least one array to concatenate")
    flat = [audio[i][j] for i, j in order]
    lens = [int(f.shape[0]) for f in flat]
    if min(lens) == 0:
        raise RuntimeError("max(): Expected reduction dim to be specified for input.numel() == 0.")
    gap = int(sr * fragment_interval)
    lib.init()
    x = torch.cat([f.reshape(-1).float() for f in flat])
    n = len(flat)
    src = np.cumsum([0] + lens[:-1])
    dst = src + np.arange(n) * gap
    table = torch.from_numpy(np.concatenate([np.stack([src, lens], 1).reshape(-1), dst]).astype(np.int64)).to(x.device)
    y = torch.empty(sum(lens) + n * gap, dtype=torch.int16, device=x.device)
    ops.fragment_int16(x, table[:2 * n].view(n, 2), table[2 * n:], max(lens), gap, y)
    return sr, y.cpu().numpy()


def _zeros(tts):
    return tts.configs.sampling_rate, np.zeros(int(tts.configs.sampling_rate), dtype=np.int16)


def _set_reference(tts, text_lang, ref_audio_path, aux_ref_audio_paths, prompt_text, prompt_lang, memo=None):
    """The language checks and the reference clip / prompt text part of `run` (tts.py:663-694) on tts.prompt_cache -> the
    prompt data to_batch takes (the cache), or None without a prompt text.  memo (run_many): a dict kept across the requests
    of one call, so that each distinct clip goes through tts.set_ref_audio / tts._get_ref_spec and each prompt text through
    the text preprocessor once; a clip or text met again is restored from it into the cache as those calls would leave it."""
    cfg = tts.configs
    no_prompt_text = prompt_text in [None, ""]
    assert text_lang in cfg.languages
    if not no_prompt_text:
        assert prompt_lang in cfg.languages
    cache = tts.prompt_cache
    if ref_audio_path in [None, ""] and (cache["prompt_semantic"] is None or cache["refer_spec"] in [None, []]):
        raise ValueError("ref_audio_path cannot be empty")
    if ref_audio_path is not None and ref_audio_path != cache["ref_audio_path"]:
        if not os.path.exists(ref_audio_path):
            raise ValueError(f"{ref_audio_path} not exists")
        if memo is not None and ref_audio_path in memo["ref"]:
            cache["prompt_semantic"], spec = memo["ref"][ref_audio_path]
            if cache["refer_spec"] in [[], None]:
                cache["refer_spec"] = [spec]
            else:
                cache["refer_spec"][0] = spec
            cache["ref_audio_path"] = ref_audio_path
        else:
            tts.set_ref_audio(ref_audio_path)
            if memo is not None:
                memo["ref"][ref_audio_path] = (cache["prompt_semantic"], cache["refer_spec"][0])
    aux_ref_audio_paths = aux_ref_audio_paths if aux_ref_audio_paths is not None else []
    paths = set(aux_ref_audio_paths) & set(cache["aux_ref_audio_paths"])
    if not (len(list(paths)) == len(aux_ref_audio_paths) == len(cache["aux_ref_audio_paths"])):
        cache["aux_ref_audio_paths"] = aux_ref_audio_paths
        cache["refer_spec"] = [cache["refer_spec"][0]]
        for path in aux_ref_audio_paths:
            if path in [None, ""] or not os.path.exists(path):
                continue
            if memo is None:
                cache["refer_spec"].append(tts._get_ref_spec(path))
                continue
            if path not in memo["aux"]:
                memo["aux"][path] = tts._get_ref_spec(path)
            cache["refer_spec"].append(memo["aux"][path])
    if not no_prompt_text:
        prompt_text = prompt_text.strip("\n")
        if prompt_text[-1] not in SPLITS:
            prompt_text += "。" if prompt_lang != "en" else "."
        if cache["prompt_text"] != prompt_text:
            cache["prompt_text"] = prompt_text
            cache["prompt_lang"] = prompt_lang
            key = (prompt_text, prompt_lang)
            if memo is None or key not in memo["prompt"]:
                feats = tts.text_preprocessor.segment_and_extract_feature_for_text(prompt_text, prompt_lang)
                if memo is not None:
                    memo["prompt"][key] = feats
            else:
                feats = memo["prompt"][key]
            cache["phones"], cache["bert_features"], cache["norm_text"] = feats
    return None if no_prompt_text else cache


@torch.no_grad()
def run(tts, inputs):
    """`TTS.run` (tts.py:577-866) for the caller's TTS object: the same inputs, defaults and (sr, int16 ndarray) yields.
    The reference clip goes through tts.set_ref_audio / tts._get_ref_spec (whose bodies are ref_spec and prompt_semantic
    after the caller's file decoding), the text through tts.text_preprocessor; batching, AR decoding (tts.t2s_model.model),
    vocoding (tts.vits_model) and the int16 assembly run on the device.  On an exception: one second of zeros is yielded,
    both models are reloaded and the exception is raised again."""
    cfg = tts.configs
    tts.stop_flag = False
    text = inputs.get("text", "")
    text_lang = inputs.get("text_lang", "")
    ref_audio_path = inputs.get("ref_audio_path", "")
    aux_ref_audio_paths = inputs.get("aux_ref_audio_paths", [])
    prompt_text = inputs.get("prompt_text", "")
    prompt_lang = inputs.get("prompt_lang", "")
    top_k = inputs.get("top_k", 5)
    top_p = inputs.get("top_p", 1)
    temperature = inputs.get("temperature", 1)
    text_split_method = inputs.get("text_split_method", "cut0")
    batch_size = inputs.get("batch_size", 1)
    batch_threshold = inputs.get("batch_threshold", 0.75)
    speed_factor = inputs.get("speed_factor", 1.0)
    split_bucket = inputs.get("split_bucket", True)
    return_fragment = inputs.get("return_fragment", False)
    fragment_interval = inputs.get("fragment_interval", 0.3)
    seed = inputs.get("seed", -1)
    set_seed(-1 if seed in ["", None] else seed)
    parallel_infer = inputs.get("parallel_infer", True)
    repetition_penalty = inputs.get("repetition_penalty", 1.35)

    t2s = tts.t2s_model.model
    t2s.infer_panel = t2s.infer_panel_batch_infer if parallel_infer else t2s.infer_panel_naive_batched
    if return_fragment or speed_factor != 1.0:
        split_bucket = False
    fragment_interval = max(fragment_interval, 0.01)
    no_prompt_text = prompt_text in [None, ""]
    prompt_data = _set_reference(tts, text_lang, ref_audio_path, aux_ref_audio_paths, prompt_text, prompt_lang)
    cache = tts.prompt_cache

    # text front end (tts.py:697-747)
    if not return_fragment:
        data = tts.text_preprocessor.preprocess(text, text_lang, text_split_method)
        if len(data) == 0:
            yield _zeros(tts)
            return
        data, batch_index_list = to_batch(data, prompt_data, batch_size, batch_threshold, split_bucket, cfg.device)
    else:
        texts = tts.text_preprocessor.pre_seg_text(text, text_lang, text_split_method)
        data = [texts[i:i + batch_size] for i in range(0, len(texts), batch_size)]

        def make_batch(batch_texts):
            batch_data = []
            for t in batch_texts:
                phones, bert_features, norm_text = tts.text_preprocessor.segment_and_extract_feature_for_text(t, text_lang)
                if phones is None:
                    continue
                batch_data.append({"phones": phones, "bert_features": bert_features, "norm_text": norm_text})
            if len(batch_data) == 0:
                return None
            return to_batch(batch_data, prompt_data, batch_size, batch_threshold, False, cfg.device)[0][0]

    try:
        audio = []
        upsample_rate = math.prod(tts.vits_model.upsample_rates)
        for item in data:
            if return_fragment:
                item = make_batch(item)
                if item is None:
                    continue
            batch_phones = item["phones"]
            prompt = None if no_prompt_text else cache["prompt_semantic"].expand(len(item["all_phones"]), -1).to(cfg.device)
            pred_semantic_list, idx_list = t2s.infer_panel(
                item["all_phones"], item["all_phones_len"], prompt, item["all_bert_features"], top_k=top_k, top_p=top_p,
                temperature=temperature, early_stop_num=cfg.hz * cfg.max_sec, max_len=item["max_len"],
                repetition_penalty=repetition_penalty)
            refer = [r.to(dtype=torch.float32, device=cfg.device) for r in cache["refer_spec"]]
            if speed_factor == 1.0:
                # one vocoder call on the bucket's concatenated codes and phones, cut at 2 * upsample_rate samples per token
                sems = [y[-idx:] for y, idx in zip(pred_semantic_list, idx_list)]
                wave = tts.vits_model.decode(torch.cat(sems).unsqueeze(0).unsqueeze(0).to(cfg.device),
                                             torch.cat(batch_phones).unsqueeze(0).to(cfg.device), refer,
                                             speed=speed_factor).detach()[0, 0, :]
                ends = np.cumsum([0] + [s.shape[0] * 2 * upsample_rate for s in sems]).tolist()
                batch_audio_fragment = [wave[ends[i]:ends[i + 1]] for i in range(len(sems))]
            else:
                batch_audio_fragment = [
                    tts.vits_model.decode(pred_semantic_list[i][-idx:].unsqueeze(0).unsqueeze(0),
                                          batch_phones[i].unsqueeze(0).to(cfg.device), refer, speed=speed_factor).detach()[0, 0, :]
                    for i, idx in enumerate(idx_list)]
            if return_fragment:
                yield audio_postprocess([batch_audio_fragment], cfg.sampling_rate, None, speed_factor, False, fragment_interval)
            else:
                audio.append(batch_audio_fragment)
            if tts.stop_flag:
                yield _zeros(tts)
                return
        if not return_fragment:
            if len(audio) == 0:
                yield _zeros(tts)
                return
            yield audio_postprocess(audio, cfg.sampling_rate, batch_index_list, speed_factor, split_bucket, fragment_interval)
    except Exception as e:
        # the reference frees and reloads both models so that a failed call does not keep their memory
        yield _zeros(tts)
        del tts.t2s_model
        del tts.vits_model
        tts.t2s_model = None
        tts.vits_model = None
        tts.init_t2s_weights(cfg.t2s_weights_path)
        tts.init_vits_weights(cfg.vits_weights_path)
        raise e
    finally:
        empty_cache = getattr(tts, "empty_cache", None)
        if empty_cache is not None:
            empty_cache()


DECODE_ROWS = 64                                                 # rows of one decode_groups call (ops.linear_rows' limit)


def unit_seeds(n, device):
    """The noise seeds of a request's first n decoding calls as `run` draws them after its set_seed(seed): one
    torch.randint(0, 2 ** 62, (1,)) on `device` per call (Text2SemanticDecoder._run_batch) -> int64 [n] on device."""
    draws = [torch.randint(0, 2 ** 62, (1,), device=device, dtype=torch.int64) for _ in range(n)]
    return torch.cat(draws) if draws else torch.zeros(0, dtype=torch.int64, device=device)


def decode_units(batches, no_prompt_text, parallel_infer, max_rows=DECODE_ROWS):
    """The decoding calls `run` makes for one request's buckets, in order -> list of (bucket index, sentence indices in the
    bucket, eos_steps, naive): with a prompt and parallel_infer, one per bucket (infer_panel_batch_infer; EOS excluded at
    step 0), without parallel_infer one per sentence (infer_panel_naive; the first 11 steps); prompt-free, one per bucket
    (infer_panel_naive_batched; 11 steps).  A bucket of more than max_rows sentences is decoded in chunks of max_rows, one
    call each, as _decode_batch does."""
    out = []
    for k, item in enumerate(batches):
        n = len(item["all_phones"])
        if not no_prompt_text and not parallel_infer:
            out += [(k, [i], 11, True) for i in range(n)]
        else:
            out += [(k, list(range(i, min(i + max_rows, n))), 1 if not no_prompt_text else 11, False)
                    for i in range(0, n, max_rows)]
    return out


def pack_units(sizes, max_rows=DECODE_ROWS):
    """Decoding calls of sizes[i] rows -> lists of call indices, each list at most max_rows rows in all, in order."""
    packs, rows = [], max_rows
    for i, n in enumerate(sizes):
        assert 1 <= n <= max_rows
        if rows + n > max_rows:
            packs.append([])
            rows = 0
        packs[-1].append(i)
        rows += n
    return packs


def _request(tts, inputs, memo):
    """Host part of one request of run_many, in `run`'s order: seed, checks, reference clip and prompt text, text front end,
    bucketing, the noise seeds of its decoding calls -> dict of per-request state (None for no sentences)."""
    cfg = tts.configs
    g = inputs.get
    seed = g("seed", -1)
    seed = set_seed(-1 if seed in ["", None] else seed)
    prompt_text, speed = g("prompt_text", ""), g("speed_factor", 1.0)
    split_bucket = g("split_bucket", True) and speed == 1.0
    no_prompt_text = prompt_text in [None, ""]
    V = tts.t2s_model.model.vocab_size
    top_k, parallel = g("top_k", 5), g("parallel_infer", True)
    if not (top_k is None and parallel is False and not no_prompt_text):
        if top_k is None or int(top_k) != top_k or not 1 <= top_k <= V:
            raise ValueError(f"run_many: top_k must be an integer in [1, {V}], got {top_k!r}")
    prompt_data = _set_reference(tts, g("text_lang", ""), g("ref_audio_path", ""), g("aux_ref_audio_paths", []), prompt_text,
                                 g("prompt_lang", ""), memo)
    cache = tts.prompt_cache
    data = tts.text_preprocessor.preprocess(g("text", ""), g("text_lang", ""), g("text_split_method", "cut0"))
    if len(data) == 0:
        return None
    batches, bil = to_batch(data, prompt_data, g("batch_size", 1), g("batch_threshold", 0.75), split_bucket, cfg.device)
    units = decode_units(batches, no_prompt_text, parallel)
    return dict(batches=batches, bil=bil, units=units, seeds=unit_seeds(len(units), cfg.device), seed=seed, speed=speed, split_bucket=split_bucket,
                interval=max(g("fragment_interval", 0.3), 0.01), no_prompt=no_prompt_text, parallel=parallel,
                prompt=None if no_prompt_text else cache["prompt_semantic"].to(cfg.device),
                refer=[r.to(dtype=torch.float32, device=cfg.device) for r in cache["refer_spec"]],
                top_k=V if top_k is None else int(top_k), top_p=g("top_p", 1), temperature=g("temperature", 1),
                # infer_panel_batch_infer does not pass repetition_penalty on to prompt-free decoding (its default 1.35 applies)
                penalty=1.35 if (no_prompt_text and parallel) else g("repetition_penalty", 1.35))


def _group(r, unit, early_stop_num):
    """decode_groups' entry for one decoding call of request state r"""
    k, sel, eos_steps, naive = unit
    item = r["batches"][k]
    rows = [item["all_phones"][i] for i in sel]
    lens = [int(x.shape[0]) for x in rows]                       # == all_phones_len
    # infer_panel_naive pads to the sentence itself, prompt-free decoding to max(max_len, longest row)
    max_len = lens[0] if naive else max([item["max_len"]] + lens) if r["no_prompt"] else item["max_len"]
    return dict(rows=rows, lens=lens,
                bert=[item["all_bert_features"][i] for i in sel], max_len=max_len, prompt=r["prompt"], eos_steps=eos_steps,
                top_k=r["top_k"], top_p=r["top_p"], temperature=r["temperature"], repetition_penalty=r["penalty"],
                early_stop_num=early_stop_num)


VOCODE_ROWS = 16                                                 # rows of one SynthesizerTrn.decode_batch call


def _vocode(tts, reqs, sems, noise=None):
    """The vocoder calls of `run` for the requests reqs[i] (None: skipped) with semantic tokens sems[i][bucket][sentence] ->
    audio[i][bucket][sentence], 1-D device waveforms.  At speed 1 each bucket is one row (its sentences' codes and phones
    concatenated, cut at 2 * prod(upsample_rates) samples per token), and the rows of every request go through
    SynthesizerTrn.decode_batch, VOCODE_ROWS at a time; at other speeds each sentence is vocoded alone by decode.  The normal
    draws of a request's vocoder call k (bucket k at speed 1, sentence k in bucket order otherwise) are keyed by (its seed, k),
    unless noise(i, k, (1, F, 192)) supplies them (tests)."""
    vits, dev = tts.vits_model, tts.configs.device
    up = math.prod(vits.upsample_rates)
    audio = [None if r is None else [None] * len(r["batches"]) for r in reqs]
    rows = []                                                    # (request, bucket, codes, phones) of the batched calls
    for i, r in enumerate(reqs):
        if r is None:
            continue
        if r["speed"] == 1.0:
            rows += [(i, k, torch.cat(sb), torch.cat(item["phones"])) for k, (item, sb) in enumerate(zip(r["batches"], sems[i]))]
            continue
        c = 0
        for k, (item, sb) in enumerate(zip(r["batches"], sems[i])):
            audio[i][k] = []
            for s_, ph in zip(sb, item["phones"]):
                shape = (1, int(2 * s_.shape[0] / r["speed"]) + 1, vits.inter_channels)
                if noise is not None:
                    z = noise(i, c, shape)
                else:
                    state = torch.tensor([r["seed"] & (2 ** 63 - 1), c << 40], dtype=torch.int64, device=dev)
                    z = ops.randn(shape, "tts.run_many.noise", device=dev, state=state)
                audio[i][k].append(vits.decode(s_.view(1, 1, -1).to(dev), ph.unsqueeze(0).to(dev), reqs[i]["refer"],
                                               speed=r["speed"], noise=z.transpose(1, 2)).detach()[0, 0, :])
                c += 1
    ges = {i: vits.ref_style(reqs[i]["refer"]) for i in sorted({row[0] for row in rows})}
    for j in range(0, len(rows), VOCODE_ROWS):
        part = rows[j:j + VOCODE_ROWS]
        zs = None if noise is None else [noise(i, k, (1, 2 * codes.shape[0], vits.inter_channels))[0] for i, k, codes, _ in part]
        waves = vits.decode_batch([codes.to(dev) for _, _, codes, _ in part], [ph.to(dev) for _, _, _, ph in part],
                                  torch.cat([ges[i] for i, _, _, _ in part]), noise=zs,
                                  noise_keys=[(reqs[i]["seed"], k) for i, k, _, _ in part])
        for (i, k, _, _), wave in zip(part, waves):
            ends = np.cumsum([0] + [s_.shape[0] * 2 * up for s_ in sems[i][k]]).tolist()
            audio[i][k] = [wave[ends[n]:ends[n + 1]] for n in range(len(sems[i][k]))]
    return audio


@torch.no_grad()
def run_many(tts, inputs_list, noise=None):
    """Several `run` requests in one call, their sentences decoded together -> (results, errors).

    inputs_list: `run`'s input dicts (same keys and defaults), all for the models of `tts`.  results: one (sr, int16 ndarray)
    per request, in input order, what `run` would yield for it alone (the whole array; run_many does not stream).  errors: a
    list of (request index, exception) for the requests rejected on the host, in input order; each of them has one second of
    zeros as its result and the others proceed.  The host checks are `run`'s (language asserts, empty or missing reference
    paths, 3 to 10 s prompt clips, which tts.set_ref_audio rejects) plus top_k in [1, V].  return_fragment raises ValueError
    for the whole call, before any device work.

    Each request goes through `run`'s host steps in input order: set_seed(seed), its reference clip (tts.set_ref_audio /
    tts._get_ref_spec once per distinct path in the call; tts.prompt_cache is left as `run` leaves it after the last request),
    tts.text_preprocessor.preprocess and to_batch, so its buckets are those of its own `run`.  The decoding calls `run` would
    make (decode_units) are packed, across requests, into Text2SemanticDecoder.decode_groups calls of at most 64 rows; the
    k-th call of a request samples with the k-th seed `run` draws after set_seed(seed) (unit_seeds), so with a fixed seed its
    tokens are those of its own `run`, whatever it shares the pass with.  Vocoding (_vocode): at speed_factor 1 every bucket
    of every request is one row of SynthesizerTrn.decode_batch, with the request's style vector and normal draws keyed by
    (seed, bucket), so a request's audio does not depend on the others; at other speeds each sentence goes through decode, one
    at a time, as in `run`.  noise(i, k, shape) replaces the draws of request i's k-th vocoder call (tests).  Every request's
    int16 array is assembled by evk_fragment_int16 into one device buffer, copied to the host once.
    Only the host checks are per request.  A failure after them (a device error, or an empty fragment, which `run` raises on
    too) fails every request of the call: both models are reloaded, as `run` does, and the exception is raised."""
    if any(inp.get("return_fragment", False) for inp in inputs_list):
        raise ValueError("run_many: return_fragment is not supported (streaming is per request: use run)")
    cfg = tts.configs
    tts.stop_flag = False
    memo = {"ref": {}, "aux": {}, "prompt": {}}
    reqs, errors = [], []
    for i, inp in enumerate(inputs_list):
        try:
            reqs.append(_request(tts, inp, memo))
        except Exception as e:                                   # noqa: BLE001 -- the request fails alone
            reqs.append(e)
            errors.append((i, e))
    try:
        t2s = tts.t2s_model.model
        early = cfg.hz * cfg.max_sec
        calls = [(i, u) for i, r in enumerate(reqs) if isinstance(r, dict) for u in range(len(r["units"]))]
        groups = [_group(reqs[i], reqs[i]["units"][u], early) for i, u in calls]
        done = {}
        for pack in pack_units([len(g["rows"]) for g in groups]):
            for p in pack:
                groups[p]["seed"] = reqs[calls[p][0]]["seeds"][calls[p][1]:calls[p][1] + 1]
            ys, fin = t2s.decode_groups([groups[p] for p in pack])
            pos = 0
            for p in pack:
                n = len(groups[p]["rows"])
                done[calls[p]] = (ys[pos:pos + n], fin[pos:pos + n])
                pos += n
        live = [r if isinstance(r, dict) else None for r in reqs]
        sems = [None] * len(reqs)
        for i, r in enumerate(live):
            if r is None:
                continue
            sems[i] = [[None] * len(item["all_phones"]) for item in r["batches"]]
            for u, (k, sel, _, naive) in enumerate(r["units"]):
                ys, fin = done[(i, u)]
                for j, y, f in zip(sel, ys, fin):
                    idx = 0 if r["no_prompt"] else (f[0] - 1 if naive else f[1])
                    sems[i][k][j] = y[-idx:]
        audio_all = _vocode(tts, live, sems, noise) if any(r is not None for r in live) else live
        flat, frags, dsts, gaps, spans, total, off = [], [], [], [], [], 0, 0
        for i, r in enumerate(live):
            if r is None:
                continue
            audio = audio_all[i]
            order = [(a, b) for a, bucket in enumerate(audio) for b in range(len(bucket))]
            if r["split_bucket"]:
                order = recovery_order([[(a, b) for b in range(len(bk))] for a, bk in enumerate(audio)], r["bil"])
            gap = int(cfg.sampling_rate * r["interval"])
            start = total
            for a, b in order:
                f = audio[a][b].reshape(-1).float()
                if f.shape[0] == 0:
                    raise RuntimeError("max(): Expected reduction dim to be specified for input.numel() == 0.")
                frags.append((off, f.shape[0]))
                off += f.shape[0]
                dsts.append(total)
                gaps.append(gap)
                flat.append(f)
                total += f.shape[0] + gap
            spans.append((i, start, total))
        results = [_zeros(tts) for _ in inputs_list]
        if flat:
            lib.init()
            x = torch.cat(flat)
            y = torch.empty(total, dtype=torch.int16, device=x.device)
            tab = torch.tensor([[a, n, d] for (a, n), d in zip(frags, dsts)], dtype=torch.int64).to(x.device)
            max_len = max(n for _, n in frags)
            # one evk_fragment_int16 call per distinct silent interval (requests choose their own)
            for gap in sorted(set(gaps)):
                sel = torch.tensor([j for j, g_ in enumerate(gaps) if g_ == gap], dtype=torch.int64, device=x.device)
                ops.fragment_int16(x, tab[sel, :2].contiguous(), tab[sel, 2].contiguous(), max_len, gap, y)
            host = y.cpu().numpy()
            for i, a, b in spans:
                results[i] = (cfg.sampling_rate, host[a:b].copy())
        return results, errors
    except Exception:
        del tts.t2s_model
        del tts.vits_model
        tts.t2s_model = None
        tts.vits_model = None
        tts.init_t2s_weights(cfg.t2s_weights_path)
        tts.init_vits_weights(cfg.vits_weights_path)
        raise
    finally:
        empty_cache = getattr(tts, "empty_cache", None)
        if empty_cache is not None:
            empty_cache()
