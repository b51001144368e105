#!/usr/bin/env python
"""Run the reference's unmodified `Normalize._name2go` (src/normalization/normalize.py:151-179) on seeded clips on the CPU,
check oracle/ssl_oracle.py against it, and write tests/golden/normalize_ssl.pt.

What is substituted, and nothing else:
  load_audio         returns the seeded clip for its path (decoding is not part of the contract)
  librosa            absent here: `librosa.resample` is ssl_oracle.resample, the closed form of resampy's kaiser_best loop at
                     ratio 1/2 (checked against the literal loop by tests/test_cpu_normalize_ssl.py)
  text front end     `_stub`s for the G2P / BERT / SynthesizerTrn imports that _name2go does not use
The reference's CNHubert (cnhubert.py) is real: transformers' HubertModel and Wav2Vec2FeatureExtractor loaded with
from_pretrained from a temporary directory holding a seeded 2-layer config, its weights and preprocessor_config.json.

Clips (ssl_oracle.clip): even and odd lengths of 0.5-0.75 s at peak 0.8, one at peak 1.6 (1 < m <= 2.2: the int16
conversion wraps), one at peak 2.5 (skipped) and one silent (NaN features: written nowhere).

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_normalize_ssl.py
"""
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hubert_oracle, ssl_oracle  # noqa: E402
from oracle.pin_against_reference import GOLD, REF, maxdiff  # noqa: E402
from oracle.ref_import import _stub  # noqa: E402

LAYERS, PARAM_SEED = 2, 61
CLIPS = [dict(name="even_0.wav", n=16000, seed=71, peak=0.8), dict(name="odd_1.wav", n=17001, seed=72, peak=0.8),
         dict(name="even_2.wav", n=24000, seed=73, peak=0.8), dict(name="wrap_3.wav", n=16999, seed=74, peak=1.6),
         dict(name="loud_4.wav", n=16000, seed=75, peak=2.5), dict(name="silent_5.wav", n=16000, seed=76, peak=0.0)]


def import_normalize(clips):
    sys.path.insert(0, REF)
    lib = _stub("librosa")
    lib.resample = lambda y, orig_sr, target_sr: (ssl_oracle.resample(y) if (orig_sr, target_sr) == (32000, 16000)
                                                  else NotImplemented)
    _stub("LangSegment")
    _stub("src.utils.config", torch=torch)            # normalize.py takes `torch` from this module's star import
    _stub("src.utils.audio", load_audio=lambda path, sr: clips[os.path.basename(path)] if sr == 32000 else None)
    _stub("src.utils.helper", random_choice=None, get_hparams_from_file=None)
    _stub("src.easevoice.module.models", SynthesizerTrn=None)
    _stub("src.easevoice.text.cleaner", clean_text=None)
    _stub("src.easevoice.text", cleaned_text_to_sequence=None, chinese=None)
    spec = importlib.util.spec_from_file_location("src.normalization.normalize", os.path.join(REF, "src/normalization/normalize.py"))
    m = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = m
    spec.loader.exec_module(m)
    assert m.CNHubert.__module__ == "src.easevoice.feature_extractor.cnhubert" and m.librosa is lib
    return m.Normalize


def write_model_dir(path, P):
    from transformers import HubertConfig, HubertModel, Wav2Vec2FeatureExtractor
    ref = HubertModel(HubertConfig(num_hidden_layers=LAYERS)).eval()
    sd = ref.state_dict()
    ref.load_state_dict(dict(P, masked_spec_embed=sd["masked_spec_embed"]))
    ref.save_pretrained(path)
    Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True,
                             return_attention_mask=False).save_pretrained(path)


def main():
    import transformers
    torch.manual_seed(0)
    m = dict(hubert_oracle.HUBERT_BASE, layers=LAYERS)
    P = hubert_oracle.init_params(hubert_oracle.param_spec(m), PARAM_SEED)
    clips = {c["name"]: ssl_oracle.clip(c) for c in CLIPS}
    Normalize = import_normalize(clips)
    gold = dict(transformers=transformers.__version__, layers=LAYERS, param_seed=PARAM_SEED, clips=CLIPS, wav={}, ssl={},
                written=[], skipped=[], failed=[])
    report = {}
    with tempfile.TemporaryDirectory() as tmp:
        model_dir, hub, w32 = (os.path.join(tmp, d) for d in ("chinese-hubert-base", "4-cnhubert", "5-wav32k"))
        for d in (hub, w32):
            os.makedirs(d)
        write_model_dir(model_dir, P)
        n = Normalize.__new__(Normalize)           # only the attributes _name2go reads (normalize.py:36-63)
        n.hubert_output_dir, n.wav_output_dir, n.normalize_ssl = hub, w32, model_dir
        n.device, n.is_half, n.maxx, n.alpha = "cpu", False, 0.95, 0.5
        for c in CLIPS:
            name = c["name"]
            ok = n._name2go(name, os.path.join(tmp, "denoised", name))
            wrote_pt = os.path.exists(os.path.join(hub, name + ".pt"))
            wrote_wav = os.path.exists(os.path.join(w32, name))
            assert wrote_pt == wrote_wav
            o = ssl_oracle.name2go(clips[name], P, m)
            if not ok:
                gold["failed"].append(name)
                assert o["status"] == ssl_oracle.NONFINITE and not wrote_pt, name
            elif not wrote_pt:
                gold["skipped"].append(name)
                assert o["status"] == ssl_oracle.SKIP, name
            else:
                gold["written"].append(name)
                from scipy.io import wavfile
                sr, wav = wavfile.read(os.path.join(w32, name))
                ssl = torch.load(os.path.join(hub, name + ".pt"), weights_only=False)
                assert sr == 32000 and wav.dtype == np.int16 and ssl.shape[:2] == (1, 768)
                assert o["status"] == ssl_oracle.OK and np.array_equal(o["wav"], wav), name
                err = maxdiff(o["ssl"], ssl)
                assert o["ssl"].shape == ssl.shape and err < 5e-5, (name, err)
                gold["wav"][name] = torch.from_numpy(wav.copy())
                gold["ssl"][name] = ssl.contiguous().clone()
                report[name] = dict(frames=int(ssl.shape[-1]), max_abs_oracle_vs_reference=err,
                                    wrapped=int((np.abs(o["wav"].astype(np.int64)) != np.abs(np.trunc(
                                        ssl_oracle.normalize(clips[name])[1]).astype(np.int64))).sum()))
    assert gold["skipped"] == ["loud_4.wav"] and gold["failed"] == ["silent_5.wav"], gold
    assert report["wrap_3.wav"]["wrapped"] > 0
    torch.save(gold, os.path.join(GOLD, "normalize_ssl.pt"))
    print(report)


if __name__ == "__main__":
    main()
