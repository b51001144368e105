#!/usr/bin/env python
"""Pin the oracle against the reference itself and (re)generate tests/golden/*.

Needs a local checkout of the reference (EVK_REFERENCE=<its directory>), CPU only.  It
  1. stubs the one missing import of the hot-path modules (librosa.filters.mel, restated in
     oracle/mel_oracle.py and cross-checked here against torchaudio's independent Slaney filterbank),
  2. imports the reference's mel_processing / models / losses unchanged,
  3. checks every oracle function against the reference on seeded inputs (asserts),
  4. writes the reference's outputs as small golden fixtures so the pin travels.

Usage:  python oracle/pin_against_reference.py
"""
import hashlib
import json
import os
import sys
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ.get("EVK_REFERENCE", "")              # a local checkout of megaease/easevoice-trainer
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import mel_oracle, s2_oracle, gpt_oracle  # noqa: E402

warnings.filterwarnings("ignore")


def import_reference():
    lib = types.ModuleType("librosa")
    filt = types.ModuleType("librosa.filters")
    filt.mel = lambda sr, n_fft, n_mels=128, fmin=0.0, fmax=None: mel_oracle.mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
    lib.filters = filt
    sys.modules["librosa"] = lib
    sys.modules["librosa.filters"] = filt
    sys.path.insert(0, REF)
    from src.easevoice.module import mel_processing, models, losses, commons  # noqa
    return mel_processing, models, losses, commons


def maxdiff(a, b):
    return float((a.double() - b.double()).abs().max())


def pin_mel(mp):
    import torchaudio
    out = {}
    for sr in (22050, 32000, 48000):
        fb = mel_oracle.mel_filterbank(sr, 2048, 128, 0.0, None)
        ta = torchaudio.functional.melscale_fbanks(1025, 0.0, sr / 2, 128, sr, norm="slaney", mel_scale="slaney").T
        d = float(np.abs(fb - ta.numpy()).max())
        assert d < 1e-6, d
        nnz = (fb != 0).sum(0)
        assert nnz.max() <= 2, "filterbank is <=2 nnz per FFT bin"
        out[f"fb_vs_torchaudio_{sr}"] = d
    y = mel_oracle.kat_sines()
    ref_mel = mp.mel_spectrogram_torch(y, 2048, 128, 22050, 640, 2048, 0.0, None)
    ref_spec = mp.spectrogram_torch(y, 2048, 22050, 640, 2048)
    o_mel = mel_oracle.mel_spectrogram(y, 2048, 128, 22050, 640, 2048, 0.0, None)
    o_spec = mel_oracle.spectrogram(y, 2048, 640, 2048)
    assert maxdiff(ref_mel, o_mel) == 0.0 and maxdiff(ref_spec, o_spec) == 0.0
    f64 = mel_oracle.mel_spectrogram_f64(y.numpy(), 2048, 128, 22050, 640, 2048, 0.0, None)
    out["oracle_f32_vs_f64_logmel_maxabs"] = float(np.abs(f64 - o_mel.numpy()).max())
    # SURVEY.md 8(c) known answers
    assert tuple(ref_mel.shape) == (8, 128, 34)
    assert abs(float(ref_mel.sum()) - (-286936.5209)) < 0.5
    assert np.allclose(ref_mel[0, :4, 0].numpy(), [0.13125055, 0.20751116, 0.28897765, 0.36968514], atol=1e-5)
    assert ref_mel[:, :, 17].argmax(1).tolist() == [8, 16, 25, 33, 41, 48, 54, 59]
    torch.save({"mel": ref_mel, "spec_b0": ref_spec[0].clone()}, os.path.join(GOLD, "mel_kat_22050.pt"))
    # native-rate random audio (config 3 flavour), two more rates
    g = torch.Generator().manual_seed(7)
    for sr, L in ((32000, 32000), (48000, 24000)):
        yy = torch.rand(3, L, generator=g) - 0.5
        mp.mel_basis.clear()   # reference caches the filterbank keyed by fmax/dtype only (mel_processing.py:80-87), not by sr
        r = mp.mel_spectrogram_torch(yy, 2048, 128, sr, 640, 2048, 0.0, None)
        o = mel_oracle.mel_spectrogram(yy, 2048, 128, sr, 640, 2048, 0.0, None)
        assert maxdiff(r, o) == 0.0
        rs = mp.spectrogram_torch(yy, 2048, sr, 640, 2048)
        assert maxdiff(mp.spec_to_mel_torch(rs, 2048, 128, sr, 0.0, None), mel_oracle.spec_to_mel(rs, 2048, 128, sr, 0.0, None)) == 0.0
        torch.save({"seed": 7, "mel": r}, os.path.join(GOLD, f"mel_rand_{sr}.pt"))
    return out


S2_CASES = {"small": (2, 48, 12, False), "ragged": (3, 56, 17, True)}
# BASELINE config 3 at the shapes bench.py times (T = 346 frames, 120 phonemes); B = 8 keeps every launch on the same
# kernel family as the benchmarked B = 16 (the dispatch thresholds are in rows = B * T) while the CPU oracle still
# finishes in about a minute on the GPU box's host cores.
S2_FULL_CASES = {"cfg3": (8, 346, 120, False), "cfg3r": (8, 346, 120, True)}


def pin_s2(models, losses, commons, cases=None):
    """Reference SynthesizerTrn/MPD (eval => dropout off, frozen VQ) vs oracle, fwd + grads."""
    res = {}
    cases = cases or S2_CASES
    m = dict(s2_oracle.S2_MODEL)
    net_g = models.SynthesizerTrn(1025, 32, n_speakers=300, **m)
    net_d = models.MultiPeriodDiscriminator(False)
    gspec, dspec = s2_oracle.generator_param_spec(), s2_oracle.discriminator_param_spec()
    sd_g, sd_d = net_g.state_dict(), net_d.state_dict()
    assert list(sd_g.keys()) == list(gspec.keys()) or set(sd_g.keys()) == set(gspec.keys()), \
        (set(sd_g) ^ set(gspec))
    for k, v in sd_g.items():
        assert tuple(v.shape) == tuple(gspec[k]), (k, v.shape, gspec[k])
    assert set(sd_d.keys()) == set(dspec.keys()), (set(sd_d) ^ set(dspec))
    for k, v in sd_d.items():
        assert tuple(v.shape) == tuple(dspec[k]), (k, v.shape, dspec[k])
    res["n_state_g"], res["n_state_d"] = len(sd_g), len(sd_d)
    res["n_params_g"] = sum(p.numel() for p in net_g.parameters())
    res["n_params_d"] = sum(p.numel() for p in net_d.parameters())

    PG = s2_oracle.init_params(gspec, 1234)
    PD = s2_oracle.init_params(dspec, 4321)
    net_g.load_state_dict(PG); net_d.load_state_dict(PD)
    net_g.eval(); net_d.eval()

    for tag, (B, T, X, ragged) in cases.items():
        wav, ssl, text, spec_len, text_len = s2_oracle.synthetic_batch(B, T, X, 99, ragged)
        spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, 640, 2048)
        g = torch.Generator().manual_seed(5)
        noise = torch.randn(B, 192, T, generator=g)
        ids = (torch.rand(B, generator=g) * (spec_len - 32 + 1)).long()

        # ---- reference with injected randomness
        orig_randn_like, orig_rss = torch.randn_like, commons.rand_slice_segments
        torch.randn_like = lambda t, **kw: noise.to(t.dtype)
        commons.rand_slice_segments = lambda x, x_lengths=None, segment_size=4: (commons.slice_segments(x, ids, segment_size), ids)
        try:
            y_hat, kl_ssl, ids_r, x_mask, z_mask, (z, z_p, m_p, logs_p, m_q, logs_q), quant = net_g(ssl, spec, spec_len, text, text_len)
        finally:
            torch.randn_like, commons.rand_slice_segments = orig_randn_like, orig_rss
        import src.easevoice.module.mel_processing as mp
        mel = mp.spec_to_mel_torch(spec, 2048, 128, 32000, 0.0, None)
        y_mel = commons.slice_segments(mel, ids, 32)
        y_hat_mel = mp.mel_spectrogram_torch(y_hat.squeeze(1), 2048, 128, 32000, 640, 2048, 0.0, None)
        y = commons.slice_segments(wav, ids * 640, 20480)
        rs, gs, _, _ = net_d(y, y_hat.detach())
        loss_disc, _, _ = losses.discriminator_loss(rs, gs)
        net_d.zero_grad(); loss_disc.backward()
        gd_ref = {k: p.grad.clone() for k, p in net_d.named_parameters()}
        rs, gs, frs, fgs = net_d(y, y_hat)
        loss_mel = torch.nn.functional.l1_loss(y_mel, y_hat_mel) * 45
        loss_kl = losses.kl_loss(z_p, logs_q, m_p, logs_p, z_mask) * 1.0
        loss_fm = losses.feature_loss(frs, fgs)
        loss_gen, _ = losses.generator_loss(gs)
        total = loss_gen + loss_fm + loss_mel + kl_ssl * 1 + loss_kl
        net_g.zero_grad(); total.backward()
        gg_ref = {k: (p.grad.clone() if p.grad is not None else None) for k, p in net_g.named_parameters()}

        # ---- oracle
        OG = {k: (v.clone().requires_grad_(True) if k not in s2_oracle.GEN_BUFFERS else v.clone()) for k, v in PG.items()}
        OD = {k: v.clone().requires_grad_(True) for k, v in PD.items()}
        o = s2_oracle.s2_losses(OG, OD, (ssl, spec, spec_len, wav, text, text_len), noise, ids)
        gd = torch.autograd.grad(o["loss_disc"], list(OD.values()), retain_graph=True)
        gd = dict(zip(OD.keys(), gd))
        gnames = [k for k in OG if k not in s2_oracle.GEN_BUFFERS]
        gg = torch.autograd.grad(o["loss_gen_all"], [OG[k] for k in gnames], allow_unused=True)
        gg = dict(zip(gnames, gg))

        def rel(a, b):
            return float((a - b).norm() / (b.norm() + 1e-12))
        checks = {
            "y_hat": rel(o["y_hat"], y_hat), "z": rel(o["z"], z), "z_p": rel(o["z_p"], z_p), "m_p": rel(o["m_p"], m_p),
            "logs_p": rel(o["logs_p"], logs_p), "m_q": rel(o["m_q"], m_q), "logs_q": rel(o["logs_q"], logs_q),
            "quantized": rel(o["quantized"], quant),
            "loss_disc": abs(float(o["loss_disc"]) - float(loss_disc)) / abs(float(loss_disc)),
            "loss_gen_all": abs(float(o["loss_gen_all"]) - float(total)) / abs(float(total)),
        }
        assert float(kl_ssl) == 0.0
        assert torch.equal(ids_r, ids)
        worst_gd = max(rel(gd[k], gd_ref[k]) for k in gd)
        if os.environ.get("PIN_VERBOSE"):
            for k in gd:
                r_ = rel(gd[k], gd_ref[k])
                if r_ > 1e-4: print("D", k, r_, float(gd_ref[k].norm()))
            for k in gnames:
                if gg[k] is not None:
                    r_ = rel(gg[k], gg_ref[k])
                    if r_ > 1e-4: print("G", k, r_, float(gg_ref[k].norm()))
        unused = sorted(k for k in gnames if gg_ref[k] is None)
        assert unused == sorted(k for k in gnames if gg[k] is None), (unused,)
        # conv_k.bias of every attention has an analytically ZERO gradient (a per-query constant added to all
        # scores cancels in the softmax); what autograd returns is rounding noise, so it is not compared.
        worst_gg = max(rel(gg[k], gg_ref[k]) for k in gnames if gg[k] is not None and not k.endswith(("conv_k.bias", "w_ks.bias")))
        checks["grad_d_worst_rel"], checks["grad_g_worst_rel"] = worst_gd, worst_gg
        print(tag, json.dumps(checks, indent=1), "unused:", unused)
        for k, v in checks.items():
            # forward quantities agree to fp32 rounding; parameter gradients pass through ~60 leaky-relu /
            # weight-norm layers where reduction order differs (fused torch._weight_norm vs composite), 3e-3 bound
            assert v < (3e-3 if k.startswith("grad_") else 2e-4), (tag, k, v)
        res[tag] = checks
        res[tag + "_unused_grads"] = unused
        # goldens: REFERENCE outputs (scalars + small slices + grad norms)
        gold = {
            "cfg": dict(B=B, T=T, X=X, ragged=ragged, batch_seed=99, noise_seed=5, g_seed=1234, d_seed=4321),
            "ids_slice": ids.tolist(), "spec_len": spec_len.tolist(), "text_len": text_len.tolist(),
            "loss_disc": float(loss_disc), "loss_gen": float(loss_gen), "loss_fm": float(loss_fm),
            "loss_mel": float(loss_mel), "loss_kl": float(loss_kl), "loss_gen_all": float(total),
            "y_hat_0_0_100_108": y_hat[0, 0, 100:108].tolist(), "y_hat_norm": float(y_hat.norm()),
            "z_p_norm": float(z_p.norm()), "m_p_norm": float(m_p.norm()), "logs_q_norm": float(logs_q.norm()),
            "codes_sum": int(s2_oracle.synthesizer_forward(PG, ssl, spec, spec_len, text, text_len, noise, ids)["codes"].sum()),
            "grad_norms_g": {k: float(gg_ref[k].norm()) for k in
                             ("dec.conv_pre.weight", "dec.ups.0.weight_v", "dec.resblocks.14.convs2.2.weight_g",
                              "enc_p.encoder_text.attn_layers.0.emb_rel_k", "enc_p.mrte.c_post.weight",
                              "enc_q.enc.in_layers.7.weight_v", "flow.flows.4.post.weight", "ref_enc.fc.fc.weight",
                              "enc_p.text_embedding.weight")},
            "grad_norms_d": {k: float(gd_ref[k].norm()) for k in
                             ("discriminators.0.convs.3.weight_v", "discriminators.0.conv_post.weight_g",
                              "discriminators.3.convs.0.weight_v", "discriminators.5.convs.4.weight_v")},
        }
        if tag in S2_FULL_CASES:       # full-size cases: the reference's norm of EVERY parameter gradient + forward slices
            gold["grad_norms_g"] = {k: float(v.norm()) for k, v in gg_ref.items() if v is not None}
            gold["grad_norms_d"] = {k: float(v.norm()) for k, v in gd_ref.items()}
            for nm, t in (("z", z), ("z_p", z_p), ("m_p", m_p), ("logs_p", logs_p), ("m_q", m_q), ("logs_q", logs_q)):
                gold[nm + "_norm"] = float(t.norm())
                gold[nm + "_b0_c5_t100_108"] = t[0, 5, 100:108].tolist()
            gold["y_hat_b1_0_4000_4008"] = y_hat[1, 0, 4000:4008].tolist()
        with open(os.path.join(GOLD, f"s2_{tag}.json"), "w") as f:
            json.dump(gold, f, indent=1)
    return res

GPT_CASES = (("small", 3, 3, 12, 20, False), ("ragged", 2, 4, 9, 17, True))
# BASELINE config 2 at the benchmarked model size: 24 layers, X = 256 phonemes, Y = 1024 semantic tokens, ragged 512..1024
GPT_FULL_CASES = (("cfg2", 24, 4, 256, 1024, True),)


def stub_torchmetrics():
    """torchmetrics is absent from this image; see pin_gpt."""
    tm = types.ModuleType("torchmetrics")
    tmc = types.ModuleType("torchmetrics.classification")

    class MulticlassAccuracy(torch.nn.Module):
        def __init__(self, num_classes, top_k=1, average="micro", multidim_average="global", ignore_index=None):
            super().__init__()
            self.top_k, self.ignore_index = top_k, ignore_index

        def forward(self, logits, target):                     # logits [B, V, T], target [B, T]
            top = logits.topk(self.top_k, dim=1).indices
            hit = (top == target.unsqueeze(1)).any(1)
            valid = target != self.ignore_index
            return (hit & valid).sum().float() / valid.sum().clamp(min=1).float()
    tmc.MulticlassAccuracy = MulticlassAccuracy
    tm.classification = tmc
    sys.modules["torchmetrics"] = tm
    sys.modules["torchmetrics.classification"] = tmc


def pin_gpt(cases=None, adam=True):
    """Stage-1 AR GPT: forward_old loss/acc/grads and ScaledAdam trajectories vs the reference classes.

    torchmetrics is absent from this image: MulticlassAccuracy(top_k=3, average="micro", ignore_index=EOS) is stubbed
    with its published semantics (a sample counts when the target is among the k largest logits; samples whose target is
    ignore_index are dropped), so the accuracy value is pinned against that restatement only.
    """
    stub_torchmetrics()
    from src.easevoice.soundstorm.auto_reg.models.t2s_model import Text2SemanticDecoder
    from src.easevoice.soundstorm.auto_reg.modules.optim import ScaledAdam
    res = {}
    for tag, nl, B, X, Y, ragged in cases or GPT_CASES:
        m = dict(gpt_oracle.GPT_MODEL, n_layer=nl)
        ref = Text2SemanticDecoder({"model": m}).eval()        # eval: dropout off (parity configuration)
        spec = gpt_oracle.gpt_param_spec(m)
        sd = ref.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items()} == spec, "state_dict contract"
        P = gpt_oracle.init_params(spec, 11 + nl)
        P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
        ref.load_state_dict(P)
        x, xl, y, yl, bert = gpt_oracle.synthetic_gpt_batch(B, X, Y, 5, ragged)
        loss_r, acc_r = ref.forward_old(x, xl, y, yl, bert)
        loss_r.backward()
        g_ref = {k: p.grad.clone() for k, p in ref.named_parameters()}
        Pq = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        loss_o, acc_o, logits, targets = gpt_oracle.forward_old(Pq, x, xl, y, yl, bert, m)
        loss_o.backward()
        dl = abs(float(loss_r) - float(loss_o)) / abs(float(loss_r))
        da = abs(float(acc_r) - float(acc_o))
        per = {k: maxdiff(g_ref[k], Pq[k].grad) / (float(g_ref[k].abs().max()) + 1e-12) for k in g_ref}
        dg = max(per.values())
        if os.environ.get("PIN_VERBOSE"):
            for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:8]:
                print("gpt", tag, k, v, float(g_ref[k].abs().max()))
        # 24 layers deep the two fp32 evaluation orders (fused F.multi_head_attention_forward path vs the restated one)
        # differ by up to ~1e-3 of a tensor's max on the tiny-gradient tensors; 3 layers: < 2e-4
        assert dl < 1e-5 and da < 1e-6 and dg < (3e-3 if nl > 8 else 2e-4), (tag, dl, da, dg)
        res[tag] = {"loss_rel": dl, "acc_abs": da, "grad_rel_max": dg}
        gold = {"model": m, "B": B, "X": X, "Y": Y, "ragged": ragged, "param_seed": 11 + nl, "batch_seed": 5,
                "alpha_text": 0.8, "alpha_audio": 1.3, "loss": float(loss_r), "acc": float(acc_r),
                "targets_sum": int(targets.sum()),
                "grad_norms": {k: float(g_ref[k].norm()) for k in
                               ("bert_proj.weight", "ar_text_position.alpha", "ar_audio_position.alpha",
                                "ar_audio_embedding.word_embeddings.weight", "h.layers.0.self_attn.in_proj_weight",
                                "h.layers.1.linear2.weight", "h.layers.1.norm2.bias", "ar_predict_layer.weight")}}
        # DPO variant (if_dpo): same weights/batch, rejected batch fixed by patching make_reject_y in the reference module
        import src.easevoice.soundstorm.auto_reg.models.t2s_model as t2s_mod
        spans = [(2 + b, 7 + 2 * b) for b in range(B)]
        ry, ryl = gpt_oracle.make_reject_given(y, spans)
        orig = t2s_mod.make_reject_y
        t2s_mod.make_reject_y = lambda y_o, y_lens: (ry, ryl)
        try:
            ref.zero_grad()
            dl_r, dacc_r = ref.forward(x, xl, y, yl, bert)
            dl_r.backward()
        finally:
            t2s_mod.make_reject_y = orig
        Pd = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        dl_o, dacc_o, l1_o, l2_o = gpt_oracle.forward_dpo(Pd, x, xl, y, yl, bert, ry, ryl, m)
        dl_o.backward()
        ddl = abs(float(dl_r) - float(dl_o)) / abs(float(dl_r))
        ddg = max(maxdiff(p.grad, Pd[k].grad) / (float(p.grad.abs().max()) + 1e-12) for k, p in ref.named_parameters())
        assert ddl < 1e-5 and ddg < (3e-3 if nl > 8 else 2e-4), (tag, ddl, ddg)
        res[tag].update(dpo_loss_rel=ddl, dpo_grad_rel_max=ddg)
        gold.update(dpo=dict(spans=spans, loss=float(dl_r), loss_1=float(l1_o), loss_2=float(l2_o), acc=float(dacc_r),
                             grad_norms={k: float(p.grad.norm()) for k, p in ref.named_parameters() if k in gold["grad_norms"]}))
        if tag == "cfg2":
            gold["grad_norms"] = {k: float(v.norm()) for k, v in g_ref.items()}
        with open(os.path.join(GOLD, f"gpt_{tag}.json"), "w") as f:
            json.dump(gold, f, indent=1)
    if not adam:
        return res
    # ---- ScaledAdam: 14 steps on a small mixed set (matrix, vector, scalar, tiny-rms tensor), lr 0.01 then 0.002
    g = torch.Generator().manual_seed(3)
    shapes = [(6, 5), (7,), (1,), (4, 3), (2, 3, 2)]
    init = [torch.randn(s, generator=g) * sc for s, sc in zip(shapes, (1.0, 0.5, 1.0, 1e-6, 4.0))]
    pr = [torch.nn.Parameter(t.clone()) for t in init]
    opt = ScaledAdam(pr, lr=0.01, betas=(0.9, 0.95), clipping_scale=2.0, parameters_names=[[f"p{i}" for i in range(len(pr))]],
                     show_dominant_parameters=False, clipping_update_period=8)
    po = [t.clone() for t in init]
    oo = gpt_oracle.ScaledAdamOracle(po, lr=0.01, clipping_update_period=8)
    traj = []
    worst = 0.0
    for it in range(30):
        grads = [torch.randn(s, generator=g) * (5.0 if it in (20, 27) else 1.0) for s in shapes]
        for p, gr in zip(pr, grads):
            p.grad = gr.clone()
        opt.step()
        oo.step(grads)
        if it == 0:
            for grp in opt.param_groups:
                grp["lr"] = 0.002
            oo.lr = 0.002
        worst = max(worst, max(maxdiff(a.data, b) / (float(a.data.abs().max()) + 1e-12) for a, b in zip(pr, po)))
        traj.append([float(p.data.double().norm()) for p in pr])
    assert worst < 2e-6, worst
    res["scaled_adam_rel_max"] = worst
    with open(os.path.join(GOLD, "scaled_adam.json"), "w") as f:
        json.dump({"shapes": shapes, "scales": [1.0, 0.5, 1.0, 1e-6, 4.0], "seed": 3, "steps": 30, "big_grad_steps": [20, 27],
                   "clipping_update_period": 8, "lr_first": 0.01, "lr_rest": 0.002, "param_norms": traj}, f, indent=1)
    return res


def pin_extract_latent(models):
    """Reference SynthesizerTrn.extract_latent (models.py:1015-1018) vs the oracle on seeded [1, 768, T] features of several
    lengths (odd T included: the stride-2 projection drops the last frame); codes must be IDENTICAL.  Writes the golden the GPU
    test and the CPU test read."""
    m = dict(s2_oracle.S2_MODEL)
    net_g = models.SynthesizerTrn(1025, 32, n_speakers=300, **m)
    PG = s2_oracle.init_params(s2_oracle.generator_param_spec(), 1234)
    net_g.load_state_dict(PG)
    net_g.eval()
    gold = {"g_seed": 1234, "ssl_seed": 77, "scale": 1.0, "cases": []}
    g = torch.Generator().manual_seed(77)
    for T in (2, 99, 346, 1001):
        ssl = torch.randn(1, 768, T, generator=g)
        with torch.no_grad():
            ref = net_g.extract_latent(ssl)
        ora = s2_oracle.extract_latent(PG, ssl)
        assert ref.shape == ora.shape == (1, 1, T // 2), (ref.shape, ora.shape)
        assert torch.equal(ref, ora), f"extract_latent codes differ at T={T}"
        gold["cases"].append({"T": T, "codes": ref[0, 0].tolist()})
    with open(os.path.join(GOLD, "extract_latent.json"), "w") as f:
        json.dump(gold, f)
    return {"cases": [c["T"] for c in gold["cases"]], "identical": True}


def pin_decode(models):
    """Reference SynthesizerTrn.decode (models.py:973-1013) vs the oracle with torch.randn_like replaced by a seeded tensor;
    writes tests/golden/decode.pt (inputs are regenerated from seeds, the golden holds the reference waveform)."""
    m = dict(s2_oracle.S2_MODEL)
    net_g = models.SynthesizerTrn(1025, 32, n_speakers=300, **m)
    PG = s2_oracle.init_params(s2_oracle.generator_param_spec(), 1234)
    net_g.load_state_dict(PG)
    net_g.eval()
    cfg = dict(g_seed=1234, seed=91, T=24, X=15, Tr=(60, 37), noise_scale=0.5)
    g = torch.Generator().manual_seed(cfg["seed"])
    codes = torch.randint(0, 1024, (1, 1, cfg["T"]), generator=g)
    text = torch.randint(0, 300, (1, cfg["X"]), generator=g)
    refers = [torch.rand(1, 1025, tr, generator=g) * 2.0 for tr in cfg["Tr"]]
    noise = torch.randn(1, 192, 2 * cfg["T"], generator=g)
    orig = torch.randn_like
    torch.randn_like = lambda t, **kw: noise.to(t.dtype)
    try:
        with torch.no_grad():
            ref = net_g.decode(codes, text, refers, noise_scale=cfg["noise_scale"])
    finally:
        torch.randn_like = orig
    with torch.no_grad():
        ora = s2_oracle.decode(PG, codes, text, refers, noise, cfg["noise_scale"])
    assert ref.shape == ora.shape == (1, 1, 2 * cfg["T"] * 640), (ref.shape, ora.shape)
    err = maxdiff(ref, ora)
    assert err < 2e-5, err
    # speed != 1: the prior is resampled to int(2T / speed) + 1 frames (models.py:246-248)
    cfg["speed"] = 1.25
    Fs = int(2 * cfg["T"] / cfg["speed"]) + 1
    noise_s = torch.randn(1, 192, Fs, generator=g)
    torch.randn_like = lambda t, **kw: noise_s.to(t.dtype)
    try:
        with torch.no_grad():
            ref_s = net_g.decode(codes, text, refers, noise_scale=cfg["noise_scale"], speed=cfg["speed"])
    finally:
        torch.randn_like = orig
    with torch.no_grad():
        ora_s = s2_oracle.decode(PG, codes, text, refers, noise_s, cfg["noise_scale"], speed=cfg["speed"])
    assert ref_s.shape == ora_s.shape == (1, 1, Fs * 640), (ref_s.shape, ora_s.shape)
    err_s = maxdiff(ref_s, ora_s)
    assert err_s < 2e-5, err_s
    torch.save({"cfg": cfg, "wave": ref.clone(), "wave_speed": ref_s.clone()}, os.path.join(GOLD, "decode.pt"))
    return {"max_abs_diff_oracle_vs_reference": err, "max_abs_diff_speed_1.25": err_s, "samples": int(ref.numel()),
            "rms": float(ref.pow(2).mean().sqrt())}


def pin_infer_panel():
    """Reference Text2SemanticDecoder.infer_panel_naive (t2s_model.py:762-867, KV cache, torch SDPA) vs the oracle (full
    recompute under the prefix-LM mask), greedy (top_k = 1: the multinomial draw is then deterministic), repetition penalty
    1.35, bounded by early_stop_num.  Token sequences must be IDENTICAL and per-step logits equal to fp32 noise.  Writes
    tests/golden/infer_panel.json (tokens, logits of selected steps, top-2 margins)."""
    stub_torchmetrics()
    import src.easevoice.soundstorm.auto_reg.models.t2s_model as t2s_mod
    m = dict(gpt_oracle.GPT_MODEL, n_layer=3)
    ref = t2s_mod.Text2SemanticDecoder({"model": m}).eval()
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), 14)
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    ref.load_state_dict(P)
    cfg = dict(n_layer=3, param_seed=14, seed=23, X=21, Yp=17, early_stop_num=40, top_k=1, repetition_penalty=1.35, temperature=1.0)
    g = torch.Generator().manual_seed(cfg["seed"])
    x = torch.randint(0, m["phoneme_vocab_size"], (1, cfg["X"]), generator=g)
    bert = torch.randn(1, 1024, cfg["X"], generator=g)
    prompts = torch.randint(0, 1024, (1, cfg["Yp"]), generator=g)
    ref_logits = []
    orig_sample = t2s_mod.sample

    def spy(logits, previous_tokens=None, **kw):
        ref_logits.append(logits.clone())
        return orig_sample(logits, previous_tokens, **kw)
    t2s_mod.sample = spy
    try:
        with torch.no_grad():
            y_ref, idx_ref = ref.infer_panel_naive(x, torch.tensor([cfg["X"]]), prompts, bert, top_k=cfg["top_k"], top_p=100,
                                                   early_stop_num=cfg["early_stop_num"], temperature=cfg["temperature"],
                                                   repetition_penalty=cfg["repetition_penalty"])
    finally:
        t2s_mod.sample = orig_sample
    tr = []
    with torch.no_grad():
        y_ora, idx_ora = gpt_oracle.infer_panel(P, x, bert, prompts, top_k=cfg["top_k"], top_p=100, early_stop_num=cfg["early_stop_num"],
                                                temperature=cfg["temperature"], repetition_penalty=cfg["repetition_penalty"], m=m, trace=tr)
    assert torch.equal(y_ref.long(), y_ora.long()) and int(idx_ref) == int(idx_ora), (y_ref, y_ora, idx_ref, idx_ora)
    assert len(tr) == len(ref_logits)
    # the spy sees the logits AFTER the idx < 11 truncation: compare on the common columns
    err = max(maxdiff(a, b[:, :a.shape[1]]) for a, b in zip(ref_logits, tr))
    assert err < 2e-4, err
    margins = []
    for a in ref_logits:
        t2 = a[0].topk(2).values
        margins.append(float(t2[0] - t2[1]))
    gold = {"cfg": cfg, "tokens": y_ref[0].tolist(), "idx": int(idx_ref), "top2_margin": margins,
            "logits_step": {str(s): tr[s][0].tolist() for s in (0, 1, 12, len(tr) - 1)}}
    with open(os.path.join(GOLD, "infer_panel.json"), "w") as f:
        json.dump(gold, f)
    return {"steps": len(tr), "generated": len(gold["tokens"]) - cfg["Yp"], "max_logit_diff_oracle_vs_reference": err,
            "min_top2_margin": min(margins)}


def pin_hubert():
    """transformers.HubertModel (the class behind the reference's CNHubert, cnhubert.py:14-33; called as
    `model.model(wav16k)["last_hidden_state"]`, normalize.py:166-168) vs oracle/hubert_oracle.py, same seeded weights:
    a 2-layer model on 1 s + the full 12-layer model on 0.5 s of audio.  Writes tests/golden/hubert.pt."""
    from transformers import HubertConfig, HubertModel
    from oracle import hubert_oracle as ho
    gold = {"cases": []}
    res = {}
    for tag, layers, L, seed in (("l2", 2, 16000, 41), ("base", 12, 8000, 42)):
        m = dict(ho.HUBERT_BASE, layers=layers)
        P = ho.init_params(ho.param_spec(m), seed)
        ref = HubertModel(HubertConfig(num_hidden_layers=layers)).eval()
        sd = ref.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items() if k != "masked_spec_embed"} == ho.param_spec(m), "state_dict contract"
        ref.load_state_dict(dict(P, masked_spec_embed=sd["masked_spec_embed"]))
        g = torch.Generator().manual_seed(seed + 100)
        wav = torch.randn(1, L, generator=g) * 0.3
        with torch.no_grad():
            o_ref = ref(wav)["last_hidden_state"]
            o_ora = ho.forward(P, wav, m)
        err = maxdiff(o_ref, o_ora)
        assert o_ref.shape == o_ora.shape and err < 5e-5, (tag, o_ref.shape, o_ora.shape, err)
        res[tag] = {"frames": int(o_ref.shape[1]), "max_abs_diff_oracle_vs_transformers": err, "out_rms": float(o_ref.pow(2).mean().sqrt())}
        gold["cases"].append({"tag": tag, "layers": layers, "L": L, "param_seed": seed, "wav_seed": seed + 100, "wav_scale": 0.3,
                              "out": o_ref.clone()})
    import transformers
    gold["transformers"] = transformers.__version__
    torch.save(gold, os.path.join(GOLD, "hubert.pt"))
    return res


def pin_ckpt_layouts(models):
    """tests/golden/ckpt_layouts.json: the state_dict layouts the reference's checkpoint consumers build (TTS.init_vits_weights:
    SynthesizerTrn without enc_q; TTS.init_t2s_weights: Text2SemanticLightningModule) and the named_parameters order by which
    its G_/D_ checkpoints index AdamW state."""
    import yaml
    from oracle import ref_import
    tts = ref_import.import_tts()
    from easevoice_trainer_b200 import configs
    from easevoice_trainer_b200.train import gpt as gpt_train
    hps = configs.load_s2_config()
    g = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                              n_speakers=hps["data"]["n_speakers"], **hps["model"])
    del g.enc_q
    config = yaml.safe_load(open(gpt_train.GPT_CONFIG_PATH))
    t2s = tts.Text2SemanticLightningModule(config, "****", is_train=False)
    rg = models.SynthesizerTrn(1025, 32, n_speakers=300, **dict(s2_oracle.S2_MODEL))
    rd = models.MultiPeriodDiscriminator(False)
    def lay(items):          # stored as digest + length + first / last entry of the canonical JSON (tests/test_cpu_ckpt_roundtrip.py)
        lst = [[k, list(v.shape)] for k, v in items]
        return dict(count=len(lst), sha256=hashlib.sha256(json.dumps(lst, separators=(",", ":")).encode()).hexdigest(), first=lst[0], last=lst[-1])
    out = dict(about="Parameter / state_dict layouts of the reference's checkpoint consumers (megaease/easevoice-trainer): the SynthesizerTrn that "
                     "TTS.init_vits_weights builds (enc_q deleted, loaded with strict=False), the Text2SemanticLightningModule that TTS.init_t2s_weights "
                     "loads strictly, and the named_parameters order of SynthesizerTrn(1025, 32, n_speakers=300) / MultiPeriodDiscriminator that "
                     "utils/path/ckpt.load_checkpoint + torch.optim.AdamW index optimizer state by. Each layout is stored as the sha256 of its canonical JSON "
                     "([[name, shape], ...] with separators (',', ':')), its length and its first and last entries.",
               vits_state=lay(g.state_dict().items()), t2s_state=lay(t2s.state_dict().items()),
               s2_g_params=lay(rg.named_parameters()), s2_d_params=lay(rd.named_parameters()))
    with open(os.path.join(GOLD, "ckpt_layouts.json"), "w") as f:
        f.write(json.dumps(out, indent=1) + "\n")
    return {k: v["count"] for k, v in out.items() if k != "about"}


def main():
    os.makedirs(GOLD, exist_ok=True)
    torch.manual_seed(0)
    if "--hubert" in sys.argv:           # only the Normalize.ssl model golden; before the librosa stub (transformers probes it)
        print(pin_hubert())
        return
    hub = pin_hubert() if len(sys.argv) == 1 else None
    mp, models, losses, commons = import_reference()
    if "--extract-latent" in sys.argv:   # only the Normalize.token golden (seconds)
        print(pin_extract_latent(models))
        return
    if "--infer-panel" in sys.argv:      # only the AR decoding golden (needs the torchmetrics stub of pin_gpt: run after it)
        stub_torchmetrics()
        print(pin_infer_panel())
        return
    if "--ckpt-layouts" in sys.argv:     # only the checkpoint-consumer layouts (seconds)
        print(pin_ckpt_layouts(models))
        return
    if "--decode" in sys.argv:           # only the TTS vocoder-call golden (seconds)
        print(pin_decode(models))
        return
    if "--full" in sys.argv:          # the benchmarked shapes (minutes of CPU time): python oracle/pin_against_reference.py --full
        mp.mel_basis.clear()
        report = {"s2": pin_s2(models, losses, commons, S2_FULL_CASES), "gpt": pin_gpt(GPT_FULL_CASES, adam=False)}
        with open(os.path.join(GOLD, "pin_report_full.json"), "w") as f:
            json.dump(report, f, indent=1)
        print("PIN OK (full-size cases)")
        return
    report = {"mel": pin_mel(mp)}
    print(json.dumps(report, indent=1))
    mp.mel_basis.clear()  # see pin_mel: the reference's filterbank cache is not keyed by sampling rate
    report["s2"] = pin_s2(models, losses, commons)
    report["gpt"] = pin_gpt()
    report["extract_latent"] = pin_extract_latent(models)
    report["decode"] = pin_decode(models)
    report["infer_panel"] = pin_infer_panel()
    report["hubert"] = hub
    with open(os.path.join(GOLD, "pin_report.json"), "w") as f:
        json.dump(report, f, indent=1)
    print("PIN OK")


if __name__ == "__main__":
    main()
