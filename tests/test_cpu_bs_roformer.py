"""CPU tests of the BS-Roformer separator: the oracle restatement (oracle/bs_roformer_oracle.py) against the outputs the
unmodified reference computed (tests/golden/bs_roformer.pt, pinned by oracle/pin_bs_roformer.py), its rotary stand-in against
the closed-form rotation, the key layout, the chunk rules of demix_track, and the host-side rejections of
easevoice_trainer_b200.bs_roformer."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import bs_roformer_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "bs_roformer.pt"), weights_only=False)


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    return float((a - b).norm() / b.norm())


def config(over):
    cfg = dict(O.SHIPPED)
    cfg.update(over)
    return cfg


@pytest.fixture(scope="module")
def R():
    from easevoice_trainer_b200 import bs_roformer
    return bs_roformer


def test_rotary_standin_closed_form():
    g = torch.Generator().manual_seed(3)
    t = torch.randn(2, 3, 37, 64, generator=g, dtype=torch.float64)
    got = O.RotaryEmbedding(64).rotate_queries_or_keys(t.float()).double()
    ref = torch.empty_like(t)
    for p in range(37):
        for i in range(32):
            a = p * 10000.0 ** (-2 * i / 64)
            c, s = math.cos(a), math.sin(a)
            x0, x1 = t[..., p, 2 * i], t[..., p, 2 * i + 1]
            ref[..., p, 2 * i] = x0 * c - x1 * s
            ref[..., p, 2 * i + 1] = x1 * c + x0 * s
    assert (got - ref).abs().max() < 2e-5


def test_param_spec_matches_golden_layout(R):
    spec = O.param_spec(config({}))
    assert [(k, tuple(v)) for k, v in spec.items()] == [(k, tuple(v)) for k, v in GOLD["keys"]]
    assert len(spec) == 675
    host = R.BSRoformer(**R.SHIPPED_CONFIG).state_dict_shapes()
    assert list(host.items()) == [(k, tuple(v)) for k, v in spec.items()]
    assert R.SHIPPED_CONFIG == O.SHIPPED


def test_oracle_small_forward_vs_golden():
    case = GOLD["small"]
    cfg = config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    out = O.forward(P, cfg, O.make_audio(case["audio_seed"], case["fwd_shape"]))
    assert rel(out[..., ::case["stride"]], case["forward"]) < 1e-5


@pytest.mark.parametrize("k", sorted(GOLD["passthrough"], key=float))
def test_oracle_passthrough_zeroed_samples(R, k):
    g = GOLD["passthrough"][k]
    n = g["n"]
    mix = O.make_audio(91, (2, n))                                          # PASS_SEED of the pin
    got = O.demix_track(lambda a: a, mix)["vocals"]
    assert np.array_equal(np.nonzero((got == 0).all(0))[0], g["zero"].numpy())
    assert np.array_equal(R.zeroed_samples(n), g["zero"].numpy())



def test_zeroed_samples_rules(R):
    c = R.CHUNK
    assert R.zeroed_samples(c).tolist() == [c - 1]
    assert R.zeroed_samples(int(0.3 * c)).tolist() == []
    assert R.zeroed_samples(3 * c + 5).tolist() == [0, c, 2 * c, 3 * c]
    z = R.zeroed_samples(int(5.5 * c)).tolist()
    assert z[:3] == [0, c - 1, c] and z[-2:] == [4 * c, 5 * c] and len(z) == 10


def test_oracle_small_demix_vs_golden():
    case = GOLD["small"]
    cfg = config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    mix = O.make_audio(case["audio_seed"] + 100, (2, int(case["demix_chunks"] * O.CHUNK)))
    got = O.demix_track(lambda a: O.forward(P, cfg, a), mix)["vocals"]
    idx = case["demix_idx"].numpy()
    assert rel(got[:, idx], case["demix"]) < 1e-5
    assert np.array_equal(np.nonzero((got == 0).all(0))[0], case["demix_zero"].numpy())


@pytest.mark.parametrize("over,msg", [
    (dict(dim_head=32), "dim_head"),
    (dict(linear_transformer_depth=1), "linear_transformer_depth"),
    (dict(num_stems=2), "num_stems"),
    (dict(stft_n_fft=2000, stft_win_length=2000), "power of two"),
    (dict(stft_win_length=1024), "stft_win_length"),
    (dict(freqs_per_bands=(2, 2, 1020)), "freqs_per_bands"),
])
def test_constructor_rejections(R, over, msg):
    with pytest.raises(ValueError, match=msg):
        R.BSRoformer(**config(over))


def _small(R):
    cfg = config(dict(dim=16, depth=1, heads=1))
    return cfg, R.BSRoformer(**cfg)


def test_load_state_dict_rules(R):
    cfg, m = _small(R)
    P = O.init_params(O.param_spec(cfg), 5)
    m.load_state_dict({k: v.half() for k, v in P.items()})                  # fp16 weights load
    with pytest.raises(ValueError, match="missing"):
        m.load_state_dict({k: v for k, v in P.items() if k != "final_norm.gamma"})
    with pytest.raises(ValueError, match="unexpected"):
        m.load_state_dict(dict(P, extra=torch.zeros(1)))
    bad = dict(P)
    bad["final_norm.gamma"] = torch.ones(17)
    with pytest.raises(ValueError, match="shape"):
        m.load_state_dict(bad)
    freqs = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    m.load_state_dict(dict(P, **{"layers.0.0.layers.0.0.rotary_embed.freqs": freqs}))
    with pytest.raises(ValueError, match="rotary"):
        m.load_state_dict(dict(P, **{"layers.0.0.layers.0.0.rotary_embed.freqs": freqs * 2}))


def test_forward_input_errors_before_gpu_work(R):
    cfg, m = _small(R)
    with pytest.raises(ValueError, match="CUDA"):
        m.forward(torch.zeros(1, 2, 4096))


def _rotary_keys(cfg):
    """the `rotary_embed.freqs` entries a checkpoint saved with rotary_embedding_torch installed holds, one per attention"""
    freqs = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    return {k.replace("to_qkv.weight", "rotary_embed.freqs"): freqs.clone() for k in O.param_spec(cfg) if k.endswith(".to_qkv.weight")}


def test_documented_separate_mdxc_swap(R, tmp_path):
    """SeparateMDXC.__init__ -> BSRoformer.from_pretrained(path, device); SeparateMDXC.separate first calls model.eval()"""
    cfg = config({})
    P = O.init_params(O.param_spec(cfg), 81)
    P.update(_rotary_keys(cfg))
    path = tmp_path / "bs_roformer.ckpt"
    torch.save({k: v.half() for k, v in P.items()}, path)
    m = R.BSRoformer.from_pretrained(str(path), device="cpu")
    assert m.eval() is m
    assert (m.dim, m.depth, m.heads, m.bands, m.hop, m.S) == (512, 12, 8, cfg["freqs_per_bands"], 441, 2)
    # folded operands: to_qkv + to_gates with the attention RMSNorm's gamma * sqrt(dim) in its columns, on the host
    q = "layers.0.0.layers.0"
    w = m.host_w[q + ".qkvg"]
    g = P[q + ".0.norm.gamma"].half().float() * 512 ** 0.5
    assert w.device.type == "cpu" and w.shape == (1544, 512)
    assert torch.allclose(w[:1536], P[q + ".0.to_qkv.weight"].half().float() * g, rtol=1e-6, atol=0)
    assert torch.allclose(w[1536:], P[q + ".0.to_gates.weight"].half().float() * g, rtol=1e-6, atol=0)
    assert len(m.host_w) == 24 * 4 + 62 + 62 * 2 and len(m.bias) == 24 * 3 + 62 + 62 * 2   # qkvg, out, ff1, ff2; band; mask MLP


def test_eval_returns_model(R):
    cfg, m = _small(R)
    assert m.eval() is m
