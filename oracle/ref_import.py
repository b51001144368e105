"""Golden-data infrastructure (oracle/pin_against_reference.py --ckpt-layouts): import pieces of the UNMODIFIED reference
from the local checkout of it that EVK_REFERENCE names.  No test imports this module.

The reference's inference module drags in the whole text front end (LangSegment, pypinyin, g2p, ffmpeg, HuBERT, Lightning);
only its checkpoint *consumers* are needed here, so the sibling modules that do not take part in weight loading are
replaced by empty stand-ins before `src/easevoice/inference/tts.py` is executed as it is.
"""
import importlib
import importlib.machinery
import os
import sys
import types

import torch

REF = os.environ.get("EVK_REFERENCE", "")


def available():
    return os.path.isdir(os.path.join(REF, "src"))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__path__ = []
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def import_hot_path():
    """-> (mel_processing, models, losses, commons) of the reference (see oracle/pin_against_reference.py)."""
    from oracle import pin_against_reference as pin
    mods = pin.import_reference()
    # the reference has its own top-level `tests` package: keep it BEHIND this repo on sys.path (spawned workers of
    # later tests re-import `tests.*` by name)
    while REF in sys.path:
        sys.path.remove(REF)
    sys.path.append(REF)
    for n in ("librosa", "librosa.filters"):
        sys.modules[n].__spec__ = importlib.machinery.ModuleSpec(n, None)
    return mods


def import_tts():
    """-> the reference's src.easevoice.inference.tts module (TTS.init_vits_weights / init_t2s_weights are the consumers
    of the exported checkpoints, inference/tts.py:265-315)."""
    import_hot_path()
    if "src.easevoice.inference.tts" in sys.modules:
        return sys.modules["src.easevoice.inference.tts"]
    pkg = _stub("src.easevoice.inference")
    pkg.__path__ = [os.path.join(REF, "src", "easevoice", "inference")]
    _stub("src.easevoice.inference.preprocessor", TextPreprocessor=object)
    _stub("src.easevoice.inference.segmentation", SPLITS=set())
    _stub("src.utils.audio", load_audio=None)
    _stub("src.easevoice.feature_extractor.cnhubert", CNHubert=object)
    _stub("ffmpeg")
    _stub("inflect", ten=None)
    _stub("pytorch_lightning", LightningModule=torch.nn.Module)
    try:
        import matplotlib  # noqa: F401
    except ImportError:                           # lr_schedulers.py:6 imports pyplot for a plotting helper only
        mpl = _stub("matplotlib")
        mpl.pyplot = _stub("matplotlib.pyplot")
    if "torchmetrics" not in sys.modules:
        class MulticlassAccuracy(torch.nn.Module):
            def __init__(self, *a, **k):
                super().__init__()
        tmc = _stub("torchmetrics.classification", MulticlassAccuracy=MulticlassAccuracy)
        _stub("torchmetrics", classification=tmc)
    return importlib.import_module("src.easevoice.inference.tts")
