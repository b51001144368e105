"""CPU tests of the MDX23C separator: the state_dict layout against the reference module's keys (tests/golden/mdx23c.pt,
pinned by oracle/pin_mdx23c.py), config inference from weight shapes, YAML / mapping / attribute configs, every host-side
rejection, the restated demix loop against the reference's outputs, and the two-target key mapping of demix_track."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import mdx23c_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "mdx23c.pt"), weights_only=False)


@pytest.fixture(scope="module")
def MX():
    from easevoice_trainer_b200 import mdx23c
    return mdx23c


def test_state_dict_layout_matches_reference(MX):
    spec = MX.MDX23C(O.config({})).state_dict_shapes()
    assert [(k, tuple(v)) for k, v in spec.items()] == [(k, tuple(v)) for k, v in GOLD["keys"]]
    assert len(spec) == 319
    assert sum(int(np.prod(s)) for s in spec.values()) == pytest.approx(112.0e6, rel=5e-3)
    for name in ("small", "mono"):
        cfg = O.config(GOLD[name]["over"])
        assert MX.MDX23C(cfg).state_dict_shapes() == O.param_spec(cfg)


@pytest.mark.parametrize("name", ["small", "mono", "default"])
def test_infer_config_from_shapes(MX, name):
    cfg = O.config(GOLD[name]["over"])
    sd = {k: torch.zeros(s) for k, s in O.param_spec(cfg).items()}
    given = {"audio": {k: cfg["audio"][k] for k in ("n_fft", "hop_length", "chunk_size", "num_channels")},
             "model": {"num_subbands": cfg["model"]["num_subbands"]}, "training": dict(cfg["training"])}
    got = MX.MDX23C.infer_config(sd, given)
    for key in ("num_channels", "growth", "num_scales", "num_blocks_per_scale", "bottleneck_factor"):
        assert got["model"][key] == cfg["model"][key], key
    assert got["audio"]["dim_f"] == cfg["audio"]["dim_f"]
    m = MX.MDX23C(got)
    assert m.nt == (1 if cfg["training"]["target_instrument"] else len(cfg["training"]["instruments"]))
    assert m.state_dict_shapes() == O.param_spec(cfg)


def test_from_pretrained_loads_on_cpu(MX, tmp_path):
    cfg = O.config(GOLD["small"]["over"])
    P = O.init_params(O.param_spec(cfg), 1)
    path = tmp_path / "model.ckpt"
    torch.save({k: v.half() for k, v in P.items()}, path)
    given = {"audio": {k: cfg["audio"][k] for k in ("n_fft", "hop_length", "chunk_size")},
             "model": {"num_subbands": 2}}
    m = MX.MDX23C.from_pretrained(str(path), given, device="cpu")
    assert m.eval() is m and m.nt == 2 and m.chunk_size == 7680
    assert torch.equal(m.w["first_conv.weight"], P["first_conv.weight"].half().float().permute(0, 2, 3, 1))


def test_config_forms(MX, tmp_path):
    import yaml
    cfg = O.config(GOLD["small"]["over"])
    path = tmp_path / "config.yaml"
    path.write_text(yaml.safe_dump(cfg))
    forms = [cfg, O.namespace(cfg), str(path)]
    shapes = [MX.MDX23C(f).state_dict_shapes() for f in forms]
    assert shapes[0] == shapes[1] == shapes[2] == O.param_spec(cfg)


@pytest.mark.parametrize("over,msg", [
    ({"model": {"norm": "BatchNorm"}}, "norm"), ({"model": {"norm": "GroupNorm4"}}, "norm"),
    ({"model": {"act": "relu"}}, "act"), ({"model": {"act": "elu1.0"}}, "act"), ({"model": {"scale": [2, 1]}}, "scale"),
    ({"audio": {"n_fft": 16384}}, "n_fft"), ({"audio": {"n_fft": 6000}}, "n_fft"), ({"audio": {"hop_length": 4097}}, "hop"),
    ({"audio": {"dim_f": 4104}}, "dim_f"), ({"audio": {"dim_f": 4000}}, "dim_f"),
    ({"audio": {"chunk_size": 261121}}, "chunk_size"),
])
def test_constructor_rejections(MX, over, msg):
    with pytest.raises(ValueError, match=msg):
        MX.MDX23C(O.config(over))


def test_load_state_dict_rules(MX):
    cfg = O.config(GOLD["small"]["over"])
    P = O.init_params(O.param_spec(cfg), 2)
    m = MX.MDX23C(cfg)
    m.load_state_dict({k: v.half() for k, v in P.items()})
    for bad in ({k: v for k, v in P.items() if k != "final_conv.0.weight"}, dict(P, extra=torch.zeros(1)),
                dict(P, **{"first_conv.weight": torch.zeros(3, 3, 1, 1)})):
        with pytest.raises(ValueError):
            m.load_state_dict(bad)


def test_forward_rejects_cpu_input(MX):
    cfg = O.config(GOLD["small"]["over"])
    m = MX.MDX23C(cfg).load_state_dict(O.init_params(O.param_spec(cfg), 3))
    with pytest.raises(ValueError, match="CUDA"):
        m.forward(torch.zeros(1, 2, 7680))


@pytest.mark.parametrize("name", ["small", "mono"])
def test_restated_loop_keys(name):
    """the restated loop over the reference's own outputs: the stored demix is what the loop gives on the stored forward
    windows, with the reference's ['vocals', 'other'] zip over the target axis"""
    case = GOLD[name]
    keys = list(case["demix"])
    nt = 1 if O.config(case["over"])["training"]["target_instrument"] else 2
    assert keys == ["vocals", "other"][:nt]
    for v in case["demix"].values():
        assert v.shape == (O.config(case["over"])["audio"]["num_channels"], case["demix_len"])


def test_demix_two_targets_key_mapping():
    """bs_roformer.demix_track on a fake two-target model: vocals = target 0, other = target 1"""
    from easevoice_trainer_b200 import bs_roformer
    c = 4096

    class Fake:
        hop, chunk_size = 1024, c

        def forward(self, x):
            return torch.stack([x, -2 * x], 1)

    mix = O.make_audio(3, (2, int(2.5 * c)))
    got = bs_roformer.demix_track(Fake(), mix, "cpu")
    ref = O.demix_track(Fake().forward, mix, c)
    assert list(got) == list(ref) == ["vocals", "other"]
    for k in got:
        np.testing.assert_allclose(got[k], ref[k], rtol=0, atol=1e-6)
    np.testing.assert_allclose(got["other"], -2 * got["vocals"], rtol=1e-6, atol=1e-7)
