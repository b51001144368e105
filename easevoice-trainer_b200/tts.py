"""Voice-clone synthesis: the computing parts of the reference's `TTS` class (src/easevoice/inference/tts.py) on this library.

The caller keeps its `TTS` object, its `TextPreprocessor` (G2P stays on the host) and its file decoding (`load_audio`,
`librosa.load`); its models are this library's `models.SynthesizerTrn`, `models_gpt.Text2SemanticDecoder`,
`hubert.CNHubert` and `bert.BertModel` (INTEGRATION §3).  Each function here replaces one method body:

  ref_spec          `_get_ref_spec` after `load_audio`: the reference clip's linear spectrogram on the device
  prompt_semantic   `_set_prompt_semantic` after `librosa.load`: HuBERT features and semantic tokens of the reference clip
  to_batch          `to_batch`: sentences grouped into buckets of similar text length, tensors on the device
  recovery_order    `recovery_order`
  run               `run`: the whole synthesis generator
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
    assert text_lang in cfg.languages
    if not no_prompt_text:
        assert prompt_lang in cfg.languages
    cache = tts.prompt_cache
    if ref_audio_path in [None, ""] and (cache["prompt_semantic"] is None or cache["refer_spec"] in [None, []]):
        raise ValueError("ref_audio_path cannot be empty")

    # reference clip and prompt text (tts.py:663-694)
    if ref_audio_path is not None and ref_audio_path != cache["ref_audio_path"]:
        if not os.path.exists(ref_audio_path):
            raise ValueError(f"{ref_audio_path} not exists")
        tts.set_ref_audio(ref_audio_path)
    aux_ref_audio_paths = aux_ref_audio_paths if aux_ref_audio_paths is not None else []
    paths = set(aux_ref_audio_paths) & set(cache["aux_ref_audio_paths"])
    if not (len(list(paths)) == len(aux_ref_audio_paths) == len(cache["aux_ref_audio_paths"])):
        cache["aux_ref_audio_paths"] = aux_ref_audio_paths
        cache["refer_spec"] = [cache["refer_spec"][0]]
        for path in aux_ref_audio_paths:
            if path in [None, ""] or not os.path.exists(path):
                continue
            cache["refer_spec"].append(tts._get_ref_spec(path))
    if not no_prompt_text:
        prompt_text = prompt_text.strip("\n")
        if prompt_text[-1] not in SPLITS:
            prompt_text += "。" if prompt_lang != "en" else "."
        if cache["prompt_text"] != prompt_text:
            cache["prompt_text"] = prompt_text
            cache["prompt_lang"] = prompt_lang
            cache["phones"], cache["bert_features"], cache["norm_text"] = \
                tts.text_preprocessor.segment_and_extract_feature_for_text(prompt_text, prompt_lang)
    prompt_data = None if no_prompt_text else cache

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
