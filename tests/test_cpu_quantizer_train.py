"""Trainable semantic quantizer (freeze_quantizer: false) without a GPU: the CPU oracle against the reference-pinned golden
(tests/golden/s2_quantizer_train.pt, written by oracle/pin_quantizer_train.py), and the checkpoint layout of the unfrozen case."""
import os

import torch

from oracle import s2_oracle
from oracle import vq_train_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s2_quantizer_train.pt")


def _gold():
    return torch.load(GOLD, weights_only=False)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


def test_oracle_matches_reference_three_steps():
    gold = _gold()
    c, run = gold["cfg"], gold["run"]
    w, b, ssls, ups = O.pin_inputs(c)
    buf = dict(embed=torch.zeros(c["K"], c["D"]), embed_avg=torch.zeros(c["K"], c["D"]), cluster_size=torch.zeros(c["K"]),
               inited=torch.zeros(1))
    for i, (ssl, up, ref) in enumerate(zip(ssls, ups, run["steps"])):
        r = O.step(ssl, w, b, buf, up, kmeans_idx=run["kmeans_idx"])
        assert torch.equal(r["codes"], ref["codes"].reshape(r["codes"].shape)), i
        assert abs(float(r["kl_ssl"]) - float(ref["kl_ssl"])) <= 1e-5 * abs(float(ref["kl_ssl"])), i
        for k in ("embed", "embed_avg", "cluster_size"):
            assert _rel(r["buffers"][k], ref["buffers"][k]) <= 2e-5, (i, k)
        assert float(r["buffers"]["inited"]) == 1.0
        assert _rel(r["dweight"], ref["dweight"]) <= 2e-5 and _rel(r["dbias"], ref["dbias"]) <= 2e-5, i
        buf = r["buffers"]


def test_kmeans_integer_samples_bit_exact():
    """All distances and means are exact here, and 64 means drawn from 40 samples of 8 distinct points tie: the oracle's
    k-means (lowest index wins a tie) must equal the reference's bit for bit."""
    ik = _gold()["kmeans_int"]
    means, bins, _ = O.kmeans(ik["samples"], 64, 50, ik["idx"])
    assert torch.equal(means, ik["means"]) and torch.equal(bins, ik["bins"])
    assert int((bins > 0).sum()) < 64               # the tie rule decided where the duplicates went


def test_dead_code_expiry_is_inert():
    """The reference's buffers and codes were the same with threshold_ema_dead_code 0 and 2 (asserted when pinning)."""
    assert _gold()["expiry_inert"] is True


def test_unfrozen_checkpoint_loads_into_torch_adamw(tmp_path):
    """An unfrozen G_*.pth carries the codebook buffers and AdamW state for ssl_proj.*, in the layout torch.optim.AdamW
    (the reference's optimizer, loaded by its utils.load_checkpoint) accepts."""
    from easevoice_trainer_b200 import models
    from easevoice_trainer_b200.train import s2_step
    from easevoice_trainer_b200.utils import ckpt
    m = dict(s2_oracle.S2_MODEL, freeze_quantizer=False)
    net = models.SynthesizerTrn(1025, 32, n_speakers=300, **m)
    cb = "quantizer.vq.layers.0._codebook."
    assert float(net.P(cb + "inited")) == 0.0 and float(net.P(cb + "embed").abs().max()) == 0.0
    opt = s2_step.FlatAdamW(net.named_parameters(), s2_step.g_param_groups(net, 0.4), (0.8, 0.99), 1e-9,
                            frozen=() if net.freeze_quantizer is False else s2_step.FROZEN_G)
    net.P(cb + "inited").fill_(1.0)
    net.P(cb + "embed").normal_()
    off, k = opt.slots["ssl_proj.weight"]
    assert off + k <= opt.n_active                   # trained and all-reduced with the rest of the base group
    opt.flat_m[off:off + k].fill_(0.25)
    path = str(tmp_path / "G_1.pth")
    ckpt.save_checkpoint(net, opt, 1e-4, 1, path)
    ck = torch.load(path, map_location="cpu")
    assert torch.equal(ck["model"][cb + "embed"], net.P(cb + "embed")) and float(ck["model"][cb + "inited"]) == 1.0
    i = opt.names.index("ssl_proj.weight")                    # state indices follow the parameter groups' order
    assert i in ck["optimizer"]["state"] and float(ck["optimizer"]["state"][i]["exp_avg"].flatten()[0]) == 0.25
    ref = models.SynthesizerTrn(1025, 32, n_speakers=300, **m)
    groups = [dict(params=[dict(ref.named_parameters())[n] for n in ns], lr=1e-4 * s) for s, ns in s2_step.g_param_groups(ref, 0.4)]
    topt = torch.optim.AdamW(groups, 1e-4, betas=(0.8, 0.99), eps=1e-9)
    topt.load_state_dict(ck["optimizer"])
    p = dict(ref.named_parameters())["ssl_proj.weight"]
    assert torch.equal(topt.state[p]["exp_avg"], torch.full_like(p, 0.25))
    # and it resumes into a fresh model: buffers and optimizer state come back
    net2 = models.SynthesizerTrn(1025, 32, n_speakers=300, **m)
    opt2 = s2_step.FlatAdamW(net2.named_parameters(), s2_step.g_param_groups(net2, 0.4), (0.8, 0.99), 1e-9)
    ckpt.load_checkpoint(path, net2, opt2)
    assert torch.equal(net2.P(cb + "embed"), net.P(cb + "embed")) and not net2.codebook_needs_init()
    assert torch.equal(opt2.flat_m[off:off + k], opt.flat_m[off:off + k])
