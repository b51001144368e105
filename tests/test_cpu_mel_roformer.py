"""CPU tests of the Mel-Band Roformer separator: the band tables of easevoice_trainer_b200.mel_band_roformer against the ones
the unmodified reference built (tests/golden/mel_roformer.pt, pinned by oracle/pin_mel_roformer.py) and against the oracle's
restatement of the reference's steps, the state_dict layout, the configuration inferred from weight shapes, the oracle
against the reference's outputs, and every host-side rejection."""
import os

import numpy as np
import pytest
import torch

from oracle import mel_roformer_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "mel_roformer.pt"), weights_only=False)


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    return float((a - b).norm() / b.norm())


def config(over):
    cfg = dict(O.DEFAULT)
    cfg.update(over)
    return cfg


@pytest.fixture(scope="module")
def M():
    from easevoice_trainer_b200 import mel_band_roformer
    return mel_band_roformer


def _check_tables(M, sr, n_fft, nb, fi, per_band, per_bin):
    bins, band_off, cover, cover_off = M.band_tables(sr, n_fft, nb)
    assert np.array_equal(bins, np.asarray(fi)) and bins.dtype == np.int32
    assert np.array_equal(np.diff(band_off), np.asarray(per_band))
    assert np.array_equal(np.diff(cover_off), np.asarray(per_bin))
    # cover lists, for every bin, the slots holding it, in ascending slot (= band) order
    for f in range(n_fft // 2 + 1):
        slots = cover[cover_off[f]:cover_off[f + 1]]
        assert (bins[slots] == f).all() and (np.diff(slots) > 0).all()
    assert np.array_equal(np.sort(cover), np.arange(len(bins)))


@pytest.mark.parametrize("key", sorted(GOLD["tables"]))
def test_band_tables_vs_reference(M, key):
    g = GOLD["tables"][key]
    _check_tables(M, *key, g["freq_indices"], g["per_band"], g["per_bin"])
    st = np.stack([2 * g["freq_indices"].numpy(), 2 * g["freq_indices"].numpy() + 1], 1).reshape(-1)
    assert np.array_equal(st, g["stereo_freq_indices"].numpy())      # the reference's interleave 2 f + s


@pytest.mark.parametrize("sr,n_fft,nb", [(44100, 2048, 60), (44100, 4096, 60), (44100, 2048, 16), (48000, 1024, 48),
                                         (16000, 512, 40), (44100, 256, 8), (32000, 2048, 100)])
def test_band_tables_vs_oracle(M, sr, n_fft, nb):
    fi, per_band, per_bin = O.band_tables(sr, n_fft, nb, False)
    _check_tables(M, sr, n_fft, nb, fi.numpy(), per_band.numpy(), per_bin.numpy())
    assert int(per_bin.max()) <= 2 and int(per_bin.min()) >= 1


def test_state_dict_shapes_match_reference_layout(M):
    spec = M.MelBandRoformer(**M.DEFAULT_CONFIG).state_dict_shapes()
    assert list(spec.items()) == [(k, tuple(v)) for k, v in GOLD["keys"]]
    for name in ("small", "mono"):
        cfg = config(GOLD[name]["over"])
        assert list(M.MelBandRoformer(**cfg).state_dict_shapes().items()) == [(k, tuple(v)) for k, v in O.param_spec(cfg).items()]
    assert M.DEFAULT_CONFIG == O.DEFAULT


def _zeros(cfg, rotary=False):
    sd = {k: torch.zeros(v) for k, v in O.param_spec(cfg).items()}
    if rotary:
        sd.update({k.replace("to_qkv.weight", "rotary_embed.freqs"): torch.zeros(32) for k in list(sd) if k.endswith("to_qkv.weight")})
    return sd


@pytest.mark.parametrize("name,given", [("default", {}), ("small", {}), ("mono", dict(match_input_audio_length=True)),
                                        ("wide", dict(sample_rate=48000, stft_hop_length=480))])
def test_infer_config_from_shapes(M, name, given):
    over = dict(dim=96, depth=3, heads=3, stereo=False, num_bands=48, stft_n_fft=4096, stft_win_length=4096,
                time_transformer_depth=2, freq_transformer_depth=1, mask_estimator_depth=0, sample_rate=48000,
                stft_hop_length=480) if name == "wide" else GOLD[name]["over"]
    cfg = config(over)
    got = M.MelBandRoformer.infer_config(_zeros(cfg, rotary=True), **given)
    for k in ("dim", "depth", "heads", "num_bands", "stereo", "stft_n_fft", "stft_win_length", "time_transformer_depth",
              "freq_transformer_depth", "mask_estimator_depth", "sample_rate", "stft_hop_length", "match_input_audio_length"):
        assert got[k] == cfg[k], (k, got[k], cfg[k])
    M.MelBandRoformer(**got)


def test_from_pretrained_infers_and_loads(M, tmp_path):
    cfg = config(GOLD["mono"]["over"])
    P = O.init_params(O.param_spec(cfg), 5)
    path = tmp_path / "mel_band_roformer.ckpt"
    torch.save({k: v.half() for k, v in P.items()}, path)
    m = M.MelBandRoformer.from_pretrained(str(path), device="cpu", match_input_audio_length=True)
    assert (m.dim, m.depth, m.heads, m.num_bands, m.n_fft, m.hop, m.S, m.mask_depth, m.t_depth, m.f_depth) == \
        (64, 2, 1, 24, 1024, 441, 1, 1, 1, 2)
    assert m.match_input_audio_length and m.eval() is m
    # the last Transformer's output-norm gamma is folded into every mask MLP's first Linear; the others stay device vectors
    g = P["layers.1.1.norm.gamma"].half().float() * 64 ** 0.5
    w = P["mask_estimators.0.to_freqs.3.0.0.weight"].half().float()
    assert torch.allclose(m.host_w["mask.3.0"], w * g, rtol=1e-6, atol=0)
    assert sorted(k for k in m.bias if k.endswith(".norm.g")) == ["layers.0.0.norm.g", "layers.0.1.norm.g", "layers.1.0.norm.g"]


def test_infer_config_rejects_inconsistent_weights(M):
    cfg = config(GOLD["small"]["over"])
    sd = _zeros(cfg)
    sd["band_split.to_features.5.0.gamma"] = torch.zeros(sd["band_split.to_features.5.0.gamma"].shape[0] + 4)
    with pytest.raises(ValueError, match="match no"):
        M.MelBandRoformer.infer_config(sd)
    with pytest.raises(ValueError, match="band_split"):
        M.MelBandRoformer.infer_config({k: v for k, v in sd.items() if not k.startswith("band_split")})
    sd = _zeros(cfg)
    with pytest.raises(ValueError, match="match no"):                 # the widths of 44.1 kHz bands are not those of 16 kHz
        M.MelBandRoformer.infer_config(sd, sample_rate=16000)
    sd["layers.0.0.layers.0.0.to_qkv.weight"] = torch.zeros(3 * 2 * 32, 128)
    with pytest.raises(ValueError, match="dim_head"):
        M.MelBandRoformer(**M.MelBandRoformer.infer_config(sd))


def test_oracle_forward_vs_golden():
    for name in ("small", "mono"):
        case = GOLD[name]
        cfg = config(case["over"])
        P = O.init_params(O.param_spec(cfg), case["seed"])
        out = O.forward(P, cfg, O.make_audio(case["audio_seed"], case["fwd_shape"]))
        assert out.shape[-1] == case["forward_len"]
        assert rel(out[..., ::case["stride"]], case["forward"]) < 1e-5


@pytest.mark.parametrize("over,msg", [
    (dict(dim_head=32), "dim_head"),
    (dict(num_stems=2), "num_stems"),
    (dict(stft_n_fft=2000, stft_win_length=2000), "power of two"),
    (dict(stft_n_fft=8192, stft_win_length=8192), "power of two"),
    (dict(stft_win_length=1024), "stft_win_length"),
    (dict(stft_normalized=True), "un-normalised"),
    (dict(stft_window_fn=torch.hamming_window), "un-normalised"),
    (dict(stft_hop_length=1025), "stft_hop_length"),
    (dict(stft_n_fft=256, stft_win_length=256, stft_hop_length=64, num_bands=128), "no bins"),
    (dict(num_bands=0), "num_bands"),
    (dict(mask_estimator_depth=-1), "mask_estimator_depth"),
    (dict(dim=130), "bad sizes"),
])
def test_constructor_rejections(M, over, msg):
    with pytest.raises(ValueError, match=msg):
        M.MelBandRoformer(**config(over))


def test_uncovered_bin_rejected(M, monkeypatch):
    """the reference's assert (every bin in some band) as a ValueError: a filterbank whose column 100 is cut leaves bin 100
    out"""
    real = M.slaney_filterbank

    def cut(*a, **k):
        fb = real(*a, **k)
        fb[:, 100] = 0.0
        return fb

    monkeypatch.setattr(M, "slaney_filterbank", cut)
    with pytest.raises(ValueError, match="covered"):
        M.MelBandRoformer(**config({}))


def _small(M):
    cfg = config(dict(dim=16, depth=1, heads=1, num_bands=8))
    return cfg, M.MelBandRoformer(**cfg)


def test_load_state_dict_rules(M):
    cfg, m = _small(M)
    P = O.init_params(O.param_spec(cfg), 5)
    m.load_state_dict({k: v.half() for k, v in P.items()})                  # fp16 weights load
    with pytest.raises(ValueError, match="missing"):
        m.load_state_dict({k: v for k, v in P.items() if k != "layers.0.0.norm.gamma"})
    with pytest.raises(ValueError, match="unexpected"):
        m.load_state_dict(dict(P, **{"final_norm.gamma": torch.ones(16)}))
    bad = dict(P)
    bad["layers.0.1.norm.gamma"] = torch.ones(17)
    with pytest.raises(ValueError, match="shape"):
        m.load_state_dict(bad)
    freqs = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    m.load_state_dict(dict(P, **{"layers.0.1.layers.0.0.rotary_embed.freqs": freqs}))
    with pytest.raises(ValueError, match="rotary"):
        m.load_state_dict(dict(P, **{"layers.0.1.layers.0.0.rotary_embed.freqs": freqs * 2}))


def test_forward_input_errors_before_gpu_work(M):
    cfg, m = _small(M)
    with pytest.raises(ValueError, match="CUDA"):
        m.forward(torch.zeros(1, 2, 4096))
