"""Normalize.ssl (SURVEY 8 row f3, ssl half): the oracle restatement of `_name2go` reproduces what the reference's unmodified
method wrote (tests/golden/normalize_ssl.pt, oracle/pin_normalize_ssl.py), the closed-form 2:1 resampling taps equal resampy's
kaiser_best loop, and the host-side checks of the drop-in reject bad input before any GPU work."""
import os

import numpy as np
import pytest
import torch

from oracle import hubert_oracle, ssl_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "normalize_ssl.pt"), weights_only=False)


def test_oracle_name2go_matches_reference_golden():
    m = dict(hubert_oracle.HUBERT_BASE, layers=GOLD["layers"])
    P = hubert_oracle.init_params(hubert_oracle.param_spec(m), GOLD["param_seed"])
    written, skipped, failed = [], [], []
    for c in GOLD["clips"]:
        o = ssl_oracle.name2go(ssl_oracle.clip(c), P, m)
        {ssl_oracle.OK: written, ssl_oracle.SKIP: skipped, ssl_oracle.NONFINITE: failed}[o["status"]].append(c["name"])
        if o["status"] == ssl_oracle.OK:
            want = GOLD["wav"][c["name"]].numpy()
            assert o["wav"].dtype == np.int16 and np.array_equal(o["wav"], want), c["name"]
            assert o["ssl"].shape == GOLD["ssl"][c["name"]].shape
            assert float((o["ssl"] - GOLD["ssl"][c["name"]]).abs().max()) <= 5e-5, c["name"]
    assert (written, skipped, failed) == (GOLD["written"], GOLD["skipped"], GOLD["failed"])


def test_int16_wraps_like_x86_numpy():
    """1 < m <= 2.2 puts |a32| past 32767: the reference's astype keeps the low 16 bits of the truncated int32"""
    c = next(c for c in GOLD["clips"] if c["name"] == "wrap_3.wav")
    _, a32, _ = ssl_oracle.normalize(ssl_oracle.clip(c))
    big = np.abs(a32) > 32767
    assert big.any()
    t = np.trunc(a32[big]).astype(np.int64)
    assert np.array_equal(GOLD["wav"]["wrap_3.wav"].numpy()[big].astype(np.int64), (t + 32768) % 65536 - 32768)


@pytest.mark.parametrize("L", [301, 400])
def test_closed_form_taps_equal_literal_resampy_loop(L):
    x = np.random.default_rng(L).standard_normal(L)
    want = ssl_oracle.librosa_resample_literal(x)
    got = ssl_oracle.resample(x)
    assert want.shape == got.shape == ((L + 1) // 2,)
    assert np.abs(got - want).max() <= 1e-12
    if L % 2:
        assert got[-1] == 0.0 and want[-1] == 0.0                   # fix_length's zero, not an FIR value


def test_product_taps_equal_oracle_taps():
    from easevoice_trainer_b200 import normalize_ssl
    h, f = normalize_ssl.resample_taps()
    assert np.array_equal(h, ssl_oracle.resample_taps())
    assert f.shape == (256,) and f[0] == 0 and np.array_equal(f[1:], h[np.abs(np.arange(1, 256) - 128)].astype(np.float32))


def test_hubert_frames_and_short_rows_raise_before_gpu_work():
    from easevoice_trainer_b200 import hubert
    net = hubert.HubertModel({"num_hidden_layers": 1})
    assert [net.num_frames(n) for n in (399, 400, 719, 720, 16000)] == [0, 1, 1, 2, 49]
    for n in (400, 401, 8000, 12345, 31999):
        assert net.num_frames(n) == (n - 400) // 320 + 1
    with pytest.raises(ValueError, match="row 1"):
        net(torch.zeros(2, 1000), lengths=[1000, 399])
    with pytest.raises(ValueError, match="row 0"):
        net(torch.zeros(1, 1000), lengths=[1001])


def test_writer_rejects_empty_and_short_audio_by_name(tmp_path):
    from easevoice_trainer_b200 import hubert, normalize_ssl
    net = hubert.HubertModel({"num_hidden_layers": 1})
    for d in ("wav", "hub", "w32"):
        os.makedirs(tmp_path / d)
    (tmp_path / "list").write_text("a.wav|zh|x\nb.wav|zh|y\n", encoding="utf8")
    audio = {"a.wav": np.zeros(1600, np.float32), "b.wav": np.zeros(0, np.float32)}
    load = lambda p, sr: audio[os.path.basename(p)]  # noqa: E731
    with pytest.raises(ValueError, match="b.wav"):
        normalize_ssl.write_hubert_features(tmp_path / "list", tmp_path / "wav", tmp_path / "hub", tmp_path / "w32", net, load)
    audio["b.wav"] = np.zeros(797, np.float32)                        # 399 samples at 16 kHz
    with pytest.raises(ValueError, match="b.wav"):
        normalize_ssl.write_hubert_features(tmp_path / "list", tmp_path / "wav", tmp_path / "hub", tmp_path / "w32", net, load)
    torch.save(torch.zeros(1), tmp_path / "hub" / "b.wav.pt")           # an existing feature file: b.wav is never loaded
    (tmp_path / "list").write_text("b.wav|zh|y\na.wav|zh|x\n", encoding="utf8")
    audio["b.wav"], audio["a.wav"] = None, np.zeros(10, np.float32)
    with pytest.raises(ValueError, match="a.wav"):
        normalize_ssl.write_hubert_features(tmp_path / "list", tmp_path / "wav", tmp_path / "hub", tmp_path / "w32", net, load)
    assert not os.listdir(tmp_path / "w32")
