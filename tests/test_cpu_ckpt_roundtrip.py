"""Checkpoints written by this package are consumed by the UNMODIFIED reference (SURVEY 8b "Files out", 8f-2):
  * stage-2 export  -> TTS.init_vits_weights            (inference/tts.py:265-299: SynthesizerTrn without enc_q, strict=False)
  * stage-1 export  -> TTS.init_t2s_weights             (inference/tts.py:301-315: Text2SemanticLightningModule, strict)
  * G_/D_ resumable -> ckpt.load_checkpoint + torch.optim.AdamW.load_state_dict + ExponentialLR (sovits.py:327-376)
and reference-style optimizer states load back into the flat optimizers.  CPU only.

What those consumers expect is pinned in tests/golden/ckpt_layouts.json, recorded from the reference: the state_dict
layouts its two loaders build, and the named_parameters order by which torch.optim.AdamW indexes the optimizer state in a
G_/D_ checkpoint (oracle/pin_against_reference.py --ckpt-layouts regenerates it)."""
import hashlib
import json
import os

import pytest
import torch

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ckpt_layouts.json")))


def _layout(items):
    return [[k, list(v.shape)] for k, v in items]


def _check_layout(items, key):
    """items == the stored reference layout `key` (count, first / last entry, sha256 of the canonical JSON)."""
    lst, gold = _layout(items), GOLD[key]
    assert len(lst) == gold["count"] and lst[0] == gold["first"] and lst[-1] == gold["last"], (key, len(lst), lst[0], lst[-1])
    assert hashlib.sha256(json.dumps(lst, separators=(",", ":")).encode()).hexdigest() == gold["sha256"], key


def test_s2_export_matches_reference_vits_loader(tmp_path):
    from easevoice_trainer_b200 import configs, models
    from easevoice_trainer_b200.utils import ckpt
    hps = configs.load_s2_config()
    net_g = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                                  n_speakers=hps["data"]["n_speakers"], **hps["model"])
    before = set(os.listdir("."))
    path = ckpt.export_weights(net_g.state_dict(), hps, "rt_e1_s10", 1, 10, str(tmp_path))
    d = torch.load(path, map_location="cpu")
    ours = d["weight"]
    # strict=False in the loader: a missing or renamed key would be skipped silently, so keys and shapes must be exactly the
    # loader's (its model lists them in module order; the export keeps ours, which is the same order)
    _check_layout(ours.items(), "vits_state")
    sd = net_g.state_dict()
    for k, v in ours.items():
        assert torch.equal(v, sd[k].half()), k
    assert ours["enc_p.text_embedding.weight"].shape[0] != 322           # the loader rejects v1 models by this shape
    cfg = d["config"]
    assert cfg["data"]["sampling_rate"] == 32000 and cfg["data"]["hop_length"] == 640
    for k in ("filter_length", "win_length", "n_speakers"):
        assert k in cfg["data"], k
    assert "segment_size" in cfg["train"] and isinstance(cfg["model"], dict)
    assert set(os.listdir(".")) == before, "the temp file of save_with_torch must live next to its target, not in the CWD"


def test_gpt_export_matches_reference_t2s_loader(tmp_path):
    import yaml
    from collections import OrderedDict
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    from easevoice_trainer_b200.train import gpt as gpt_train
    config = yaml.safe_load(open(gpt_train.GPT_CONFIG_PATH))
    net = Text2SemanticDecoder(config, top_k=3)
    sd = OrderedDict(("model." + k, v.detach().clone()) for k, v in net.state_dict().items())
    _check_layout(sd.items(), "t2s_state")                               # load_state_dict(strict=True) in the loader
    assert "max_sec" in config["data"]


def _ref_optim_g(net_g, lr=1e-4, low=0.4):
    """The reference's optimizer of G (sovits.py): AdamW over four lr groups, text-side modules at lr * low."""
    te = list(map(id, net_g.enc_p.text_embedding.parameters()))
    et = list(map(id, net_g.enc_p.encoder_text.parameters()))
    mr = list(map(id, net_g.enc_p.mrte.parameters()))
    base = [p for p in net_g.parameters() if id(p) not in te + et + mr]
    return torch.optim.AdamW([{"params": base, "lr": lr}, {"params": net_g.enc_p.text_embedding.parameters(), "lr": lr * low},
                              {"params": net_g.enc_p.encoder_text.parameters(), "lr": lr * low},
                              {"params": net_g.enc_p.mrte.parameters(), "lr": lr * low}], lr, betas=(0.8, 0.99), eps=1e-9)


def _ref_load_checkpoint(path, model, optimizer):
    """What the reference's utils/path/ckpt.load_checkpoint does with a G_/D_ file: optimizer state first, then every key of
    the model's own state_dict taken from the file with an equal shape, then a strict load."""
    d = torch.load(path, map_location="cpu")
    optimizer.load_state_dict(d["optimizer"])
    own = model.state_dict()
    for k, v in own.items():
        assert k in d["model"] and d["model"][k].shape == v.shape, k
    model.load_state_dict({k: d["model"][k] for k in own})
    return d["learning_rate"], d["iteration"]


def test_resumable_checkpoints_round_trip_with_reference_optimizer(tmp_path):
    """our G_/D_ -> the reference's loading recipe + AdamW + ExponentialLR + one optimizer step; and back."""
    from easevoice_trainer_b200 import models
    from easevoice_trainer_b200.train import s2_step
    from easevoice_trainer_b200.utils import ckpt
    from oracle import s2_oracle
    og = models.SynthesizerTrn(1025, 32, n_speakers=300, **dict(s2_oracle.S2_MODEL))
    od = models.MultiPeriodDiscriminator(False)
    opt_g = s2_step.FlatAdamW(og.named_parameters(), s2_step.g_param_groups(og, 0.4), (0.8, 0.99), 1e-9, frozen=s2_step.FROZEN_G)
    opt_d = s2_step.FlatAdamW(od.named_parameters(), [(1.0, [n for n, _ in od.named_parameters()])], (0.8, 0.99), 1e-9)
    for o in (opt_g, opt_d):
        o.set_lr(9.9e-5)
        o.flat_m.normal_(); o.flat_v.uniform_(0.1, 1.0); o.hyper[1] = 7.0
    pg, pd = os.path.join(tmp_path, "G_latest.pth"), os.path.join(tmp_path, "D_latest.pth")
    ckpt.save_checkpoint(og, opt_g, 1e-4, 3, pg)
    ckpt.save_checkpoint(od, opt_d, 1e-4, 3, pd)
    # the reference's networks index optimizer state by this parameter order: ours must have the same one
    rg = models.SynthesizerTrn(1025, 32, n_speakers=300, **dict(s2_oracle.S2_MODEL))
    rd = models.MultiPeriodDiscriminator(False)
    _check_layout(rg.named_parameters(), "s2_g_params")
    _check_layout(rd.named_parameters(), "s2_d_params")
    ropt_g, ropt_d = _ref_optim_g(rg), torch.optim.AdamW(rd.parameters(), 1e-4, betas=(0.8, 0.99), eps=1e-9)
    lr, it = _ref_load_checkpoint(pd, rd, ropt_d)
    lr, it = _ref_load_checkpoint(pg, rg, ropt_g)
    assert it == 3 and lr == 1e-4
    for (n, p), (n2, p2) in zip(rg.named_parameters(), og.named_parameters()):
        assert n == n2 and torch.equal(p.data, p2.data), n
    sched = torch.optim.lr_scheduler.ExponentialLR(ropt_g, gamma=0.999875, last_epoch=-1)   # needs 'lr' / 'initial_lr'
    sched.step()
    assert abs(ropt_g.param_groups[0]["lr"] - 9.9e-5 * 0.999875) < 1e-12
    assert abs(ropt_g.param_groups[1]["lr"] - 0.4 * 9.9e-5 * 0.999875) < 1e-12
    # state tensors landed on the right parameters (index order == reference named_parameters order)
    plist = [p for g in ropt_g.param_groups for p in g["params"]]
    idx = {id(p): i for i, p in enumerate(plist)}
    byname = dict(rg.named_parameters())
    for n in ("dec.conv_pre.weight", "enc_p.mrte.c_post.weight", "enc_q.enc.cond_layer.weight_v", "flow.flows.6.post.bias"):
        assert id(byname[n]) in idx, n
        off, k = opt_g.slots[n]
        assert torch.equal(ropt_g.state[byname[n]]["exp_avg"].reshape(-1), opt_g.flat_m[off:off + k]), n
        assert float(ropt_g.state[byname[n]]["step"]) == 7.0
    assert byname["ssl_proj.weight"] not in ropt_g.state          # never-updated parameters carry no state, as in the reference
    for p in rg.parameters():
        p.grad = torch.zeros_like(p)
    ropt_g.step()                                                 # a full torch AdamW step runs on the loaded state
    # ---- and back: a checkpoint in the reference's G_ format ({model, iteration, optimizer, learning_rate}) resumes in the flat optimizer
    rpath = os.path.join(tmp_path, "G_ref.pth")
    torch.save({"model": rg.state_dict(), "iteration": 4, "optimizer": ropt_g.state_dict(), "learning_rate": 1e-4}, rpath)
    og2 = models.SynthesizerTrn(1025, 32, n_speakers=300, **dict(s2_oracle.S2_MODEL))
    opt2 = s2_step.FlatAdamW(og2.named_parameters(), s2_step.g_param_groups(og2, 0.4), (0.8, 0.99), 1e-9, frozen=s2_step.FROZEN_G)
    _, _, _, it2 = ckpt.load_checkpoint(rpath, og2, opt2)
    assert it2 == 4 and opt2.step_count == 8
    off, k = opt2.slots["dec.conv_pre.weight"]
    assert torch.equal(opt2.flat_m[off:off + k], ropt_g.state[byname["dec.conv_pre.weight"]]["exp_avg"].reshape(-1))
    assert abs(opt2.lr_host - ropt_g.param_groups[0]["lr"]) < 1e-12


def test_frozen_parameters_are_not_updated_cpu_semantics():
    """ssl_proj never receives a gradient (models.py:911-921): it sits outside every update range, and a missing gradient
    for any other parameter is an error instead of a silent zero + weight decay."""
    from easevoice_trainer_b200 import models
    from easevoice_trainer_b200.train import s2_step
    from oracle import s2_oracle
    og = models.SynthesizerTrn(1025, 32, n_speakers=300, **dict(s2_oracle.S2_MODEL))
    opt = s2_step.FlatAdamW(og.named_parameters(), s2_step.g_param_groups(og, 0.4), (0.8, 0.99), 1e-9, frozen=s2_step.FROZEN_G)
    for n in s2_step.FROZEN_G:
        off, k = opt.slots[n]
        assert off >= opt.n_active
    assert all(g["end"] <= opt.n_active for g in opt.groups)
    assert opt.reduce_view.numel() == opt.n_active == sum(p.numel() for n, p in og.named_parameters() if n not in s2_step.FROZEN_G)
    grads = [None if n in s2_step.FROZEN_G else torch.zeros_like(p) for n, p in zip(opt.names, opt.params)]
    opt.set_grads(grads)
    grads[0] = None
    with pytest.raises(RuntimeError):
        opt.set_grads(grads)
