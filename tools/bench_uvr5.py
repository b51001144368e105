#!/usr/bin/env python
"""Benchmark the UVR5 VR separator (uvr5.py) on one stereo spectrogram of a 3-minute song (44.1 kHz, hop 480: 16 538
frames, 673 bins, the default 61968 net with seeded weights), and on the same GPU the reference's algorithm on stock PyTorch
(oracle/uvr5_oracle.py's predict, one window per call with a host copy after each, as SeparateVR.inference does):
  * fp16 weights and windows (cfg.is_half, the shipped setting), cuDNN;
  * fp32 with TF32 convolutions allowed.
Also the rate of evk_conv2d_fwd on the decoder shapes of the 61968 net at 16 windows per launch.  Prints one JSON line.

--net deecho / dereverb measures the DeEcho (nout 48) / DeReverb (nout 64) CascadedNet on the same spectrogram instead
(44 windows at roi 384): uvr5.inference with and without TTA, peak device memory, the time split of one predict between
the convolutions and the LSTM, the stg3 LSTM recurrence alone, and the reference's algorithm on stock PyTorch
(oracle/uvr5_echo_oracle.py's predict with cuDNN convolutions and LSTM, one window per call with a host copy, TTA off) in
fp16 and in fp32 with TF32 allowed.

--net roformer measures the BS-Roformer (bs_roformer.py, the shipped SeparateMDXC config with seeded weights) on a 3-minute
stereo mix at 44.1 kHz (7 938 000 samples, 23 chunks): bs_roformer.demix_track (first call and `--reps` synchronised calls),
peak device memory, device time by kernel family in a separate profiled forward of `--max-chunks` chunks, the rate of
evk_rope_attn_fwd at the time and frequency shapes of 4 chunks, and the reference's algorithm on stock PyTorch
(oracle/bs_roformer_oracle.py's forward driven by its demix_track: batches of 4, a host copy and accumulate after each, SDPA
limited to the math and memory-efficient backends as Attend does off A100) with fp16 weights and chunks under autocast, as
SeparateMDXC runs with cfg.is_half (when that does not run, the error is recorded and autocast with fp32 weights is timed
instead), and in fp32 with TF32 allowed.  Every output is also compared with one run of the same algorithm in fp32 with TF32
off.

--wave measures SeparateVR.separate from waveform to waveform on a seeded 3-minute stereo mix (7 938 000 samples at 44.1
kHz, l = 16 538 frames) with --net vr (61968, 4band_v2), deecho (nout 48) or dereverb (nout 64) (4band_v3) and --tta:
uvr5.separate_wave with a host array in and host arrays out, synchronised; the reference's host path (the oracle's librosa
restatement, which makes the numpy / scipy calls librosa makes, around uvr5.inference), split into host front end, net and
host back end; and, in a separate profiled call, the device time of the new front / back-end kernels against the net.
The parameter sets are read from tests/golden/uvr5_wave.pt.

--net melroformer measures the Mel-Band Roformer (mel_band_roformer.py, the widely distributed vocal model's configuration
with seeded weights) the same way on the same mix, with the overlapping-band kernel families (evk_band_input,
evk_melband_mask_avg) split out of the device time, and oracle/mel_roformer_oracle.py's forward as the stock PyTorch arms.
It skips the rope_attn rates, whose shapes are the BS-Roformer's.

--precision float16 | bfloat16 (with --net roformer or melroformer) adds an arm with that compute type
(set_compute_type): its demix_track calls alternate with the fp32 arm's, and it gets its own peak memory, device-time split,
rope_attn rates (evk_rope_attn_fwd_h16) and rel-L2 against the fp32 arm and against the stock PyTorch arms.
With --net vr, deecho, dereverb or mdx23c (with or without --wave) it runs the library only, with the fp32 (TF32) arm and the
16-bit arm alternating call by call on the same input (uvr5.inference on the 16 538-frame spectrogram, demix_track or
separate_wave on the 3-minute mix): call times, peak memory per arm, the device time of one profiled forward split into the
convolutions (evk_conv2d_fwd / evk_conv2d_fwd_h16, with their TFLOP/s from the layer shapes) and everything else, the rel-L2
of the 16-bit output against the fp32 arm's, and whether the 16-bit output is finite.

--net mdx23c measures MDX23C (mdx23c.py, the 8K-FFT InstVoc configuration with seeded weights) the same way on the same mix
(31 chunks of 261 120 samples): demix_track wall time and peak memory, the device time of one profiled forward of
`--max-chunks` chunks split into 3x3 convs, 2x2 down / up convs, TDF Linears, instance norms, STFT / iSTFT and the rest, the
conv FLOP rate with FLOPs computed from the layer shapes here, and oracle/mdx23c_oracle.py's forward (the reference module
restated) as the stock PyTorch arms.

Usage:  python tools/bench_uvr5.py [--net vr|deecho|dereverb|roformer|melroformer|mdx23c] [--wave] [--frames 16538] [--tta 0] [--max-windows 16]
        [--reps 3] [--precision float32|float16|bfloat16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bs_roformer_oracle as BR  # noqa: E402
from oracle import mdx23c_oracle as MX  # noqa: E402
from oracle import mel_roformer_oracle as MR  # noqa: E402
from oracle import uvr5_echo_oracle as E  # noqa: E402
from oracle import uvr5_oracle as O  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return ts


def torch_inference(P, spec, agg, data, half):
    """SeparateVR.inference's window loop on stock PyTorch: one window per predict, copied to the host after each"""
    dev = torch.device("cuda")
    Pd = {k: (v.half() if half and v.is_floating_point() else v).to(dev) for k, v in P.items()}
    x_mag = np.abs(spec)
    x_phase = np.angle(spec)
    coef = x_mag.max()
    x_pre = x_mag / coef
    n = x_pre.shape[2]
    l, r, roi = O.make_padding(n, 512, O.OFFSET)
    nw = int(np.ceil(n / roi))

    def run(l, r, nw):
        xp = np.pad(x_pre, ((0, 0), (0, 0), (l, r)))
        out = []
        with torch.no_grad():
            for i in range(nw):
                w = torch.from_numpy(xp[None, :, :, i * roi: i * roi + 512])
                w = (w.half() if half else w).to(dev)
                out.append(O.predict(Pd, w, agg)[0].float().cpu().numpy())
        return np.concatenate(out, 2)

    pred = run(l, r, nw)[:, :, :n]
    if data["tta"]:
        pred = (pred + run(l + roi // 2, r + roi // 2, nw + 1)[:, :, roi // 2:][:, :, :n]) * 0.5
    return pred * coef, x_mag, np.exp(1.0j * x_phase)


def decoder_rates(ops, B, reps=20):
    """TFLOP/s of evk_conv2d_fwd on the 3x3 decoder convolutions of the 61968 net (CUDA events over `reps` launches)"""
    out = {}
    shapes = [("stg1 dec1", 336, 512, 96, 32), ("stg3 dec1", 672, 512, 192, 64), ("stg3 dec2", 336, 256, 384, 128),
              ("stg3 dec3", 168, 128, 768, 256), ("stg3 dec4", 84, 64, 1536, 512)]
    for name, H, W, C, N in shapes:
        x = torch.randn(B, H, W, C, device="cuda")
        w = torch.randn(N, 3, 3, C, device="cuda") * 0.02
        y = torch.empty(B, H, W, N, device="cuda")
        xv, yv = ops.CLView(x), ops.CLView(y)
        for _ in range(2):
            ops.conv2d(xv, w, yv, k=3, pad=1, act=ops.C2_RELU)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.conv2d(xv, w, yv, k=3, pad=1, act=ops.C2_RELU)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = dict(ms=round(ms, 3), tflops=round(2.0 * B * H * W * N * 9 * C / ms / 1e9, 1))
    return out


def torch_echo_inference(P, lstms, spec, half):
    """SeparateVREcho.inference's window loop on stock PyTorch (cuDNN convolutions and LSTM): one window per predict,
    copied to the host after each, TTA off"""
    dev = torch.device("cuda")
    x_mag = np.abs(spec)
    x_phase = np.angle(spec)
    coef = x_mag.max()
    x_pre = x_mag / coef
    n = x_pre.shape[2]
    l, r, roi = E.make_padding(n, 512, E.OFFSET)
    xp = np.pad(x_pre, ((0, 0), (0, 0), (l, r)))
    out = []
    with torch.no_grad():
        for i in range(int(np.ceil(n / roi))):
            w = torch.from_numpy(xp[None, :, :, i * roi: i * roi + 512])
            w = (w.half() if half else w).to(dev)
            out.append(E.predict(P, w, None, 1344, lstms)[0].float().cpu().numpy())
    return np.concatenate(out, 2)[:, :, :n] * coef, x_mag, np.exp(1.0j * x_phase)


def lstm_alone(ops, reps=20):
    """CUDA-event ms of the stg3 LSTMModule pieces at N = 16 windows, T = 256, I = 336, H = 64: the recurrence alone, and
    the two projection GEMMs around it"""
    N, T, I, H = 16, 256, 336, 64
    x = torch.randn(N * T, I, device="cuda")
    w_ih, b = torch.randn(8 * H, I, device="cuda") / I ** 0.5, torch.randn(8 * H, device="cuda") * 0.1
    w_hh = (torch.rand(2, 4 * H, H, device="cuda") * 2 - 1) / H ** 0.5
    w_d, b_d = torch.randn(I, 2 * H, device="cuda") / (2 * H) ** 0.5, torch.randn(I, device="cuda") * 0.1
    g = ops.gemm_tf32(x, w_ih, bias=b).view(N, T, 8 * H)
    y = ops.lstm_bidir(g, w_hh, order="nt")
    out = {}
    for name, fn in (("recurrence_ms", lambda: ops.lstm_bidir(g, w_hh, order="nt")),
                     ("projections_ms", lambda: (ops.gemm_tf32(x, w_ih, bias=b),
                                                 ops.gemm_tf32(y.view(N * T, 2 * H), w_d, bias=b_d, act=ops.ACT_RELU)))):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = round(e0.elapsed_time(e1) / reps, 4)
    return out


def echo_main(a):
    """--net deecho / dereverb: the DeEcho (nout 48) or DeReverb (nout 64) CascadedNet at n_fft 1344"""
    assert torch.cuda.is_available(), "needs a GPU"
    from easevoice_trainer_b200 import lib, ops, uvr5
    lib.init().evk_set_precise(0)
    nout = 48 if a.net == "deecho" else 64
    P = E.init_params(E.param_spec(1344, nout), 51)
    net = uvr5.CascadedNet(1344, nout).to("cuda").load_state_dict(P)
    spec = E.make_spec(7, 673, a.frames)
    roi = 512 - 2 * net.offset
    n_win = int(np.ceil(a.frames / roi))
    res = dict(gpu=gpu_info(), net=a.net, nout=nout, frames=a.frames, windows=n_win, windows_tta=2 * n_win + 1,
               max_windows=a.max_windows)
    t = time.perf_counter()
    uvr5.inference(spec, "cuda", net, None, {"window_size": 512, "tta": False}, a.max_windows)   # allocator warm-up
    res["evk_first_call_s"] = round(time.perf_counter() - t, 3)
    for tta in (False, True):
        data = {"window_size": 512, "tta": tta}
        torch.cuda.reset_peak_memory_stats()
        ts = timed(lambda: uvr5.inference(spec, "cuda", net, None, data, a.max_windows), a.reps)
        res["evk_tta_s" if tta else "evk_s"] = [round(t, 3) for t in ts]
        res["peak_mem_gib_tta" if tta else "peak_mem_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    ops.profile_begin()
    net.predict(torch.rand(a.max_windows, 2, 673, 512, device="cuda"))
    prof = ops.profile_end()
    tot = sum(v["ms"] for v in prof.values())
    conv = [v for k, v in prof.items() if k.startswith("evk_conv2d_fwd")]
    conv_ms, conv_fl = sum(v["ms"] for v in conv), sum(v["flops"] for v in conv)
    lstm_ms = prof.get("evk_lstm_bidir_fwd", dict(ms=0.0))["ms"]
    gemm_ms = sum(v["ms"] for k, v in prof.items() if k.startswith("evk_gemm_tf32"))
    res["predict_ms_by_family"] = {k: round(v["ms"], 2) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}
    res["window_gflop_conv"] = round(conv_fl / a.max_windows / 1e9, 1)
    res["predict_split"] = dict(conv2d=round(conv_ms / tot, 3), lstm_recurrence=round(lstm_ms / tot, 4),
                                lstm_gemms=round(gemm_ms / tot, 4))
    res["conv2d_tflops_in_predict"] = round(conv_fl / conv_ms / 1e9, 1)
    res["lstm_stg3_alone"] = lstm_alone(ops)
    pred = uvr5.inference(spec, "cuda", net, None, {"window_size": 512, "tta": False}, a.max_windows)[0]

    if not a.skip_torch:
        torch.backends.cudnn.benchmark = True
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cuda.matmul.allow_tf32 = True
        for name, half in (("torch_fp16", True), ("torch_tf32", False)):
            dt = torch.float16 if half else torch.float32
            Pd = {k: (v.to(dt) if v.is_floating_point() else v).to("cuda") for k, v in P.items()}
            lstms = E.lstm_modules(Pd, "cuda", dt)
            torch_echo_inference(Pd, lstms, E.make_spec(1, 673, 600), half)             # warm-up (cuDNN algorithm choice)
            ts = timed(lambda: torch_echo_inference(Pd, lstms, spec, half), a.reps)
            res[name + "_s"] = [round(t, 3) for t in ts]
            ref = torch_echo_inference(Pd, lstms, spec, half)[0]
            res[name + "_rel_l2_vs_evk"] = float(np.linalg.norm(ref - pred) / np.linalg.norm(ref))
    print(json.dumps(res))


def rope_attn_rates(ops, reps=20, dtype=None):
    """TFLOP/s of evk_rope_attn_fwd (dtype None) or evk_rope_attn_fwd_h16 at the shapes of 4 chunks of the shipped config
    (801 frames x 62 bands, 8 heads): time axis 248 sequences of 801 tokens, frequency axis 3 204 sequences of 62 tokens
    (CUDA events over `reps` launches)"""
    B, T, F, H = 4, 801, 62, 8
    ld = 3 * H * 64 + H
    x = torch.randn(B * T * F, ld, device="cuda")
    o = torch.empty(B * T * F, H * 64, device="cuda")
    out = {}
    for name, L, geo, nseq in (("time", T, (B, T * F, F, 1, F), B * F), ("freq", F, (B * T, F, 1, 0, 1), B * T)):
        cs = torch.stack(BR.rotary_cos_sin(L), -1).contiguous().cuda()
        if dtype is None:
            fn = lambda: ops.rope_attn(x, cs, o, H, L, *geo)  # noqa: E731
        else:
            fn = lambda: ops.rope_attn_h16(x, cs, o, H, L, *geo, dtype)  # noqa: E731
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = dict(sequences=nseq, L=L, ms=round(ms, 3), tflops=round(4.0 * nseq * H * L * L * 64 / ms / 1e9, 1))
    return out


FAMILIES = (("gemm", ("evk_gconv_fwd", "evk_linear_h16")), ("attention", ("evk_rope_attn_fwd", "evk_rope_attn_fwd_h16")),
            ("norms", ("evk_row_norm", "evk_band_input")), ("stft_istft", ("evk_stft_fwd", "evk_istft")))


def torch_roformer_demix(P, cfg, mix, half, autocast, forward=BR.forward):
    """SeparateMDXC.demix_track on stock PyTorch: the oracle's forward on the GPU (half: chunks cast to fp16 as the
    reference does under cfg.is_half; the weights are whatever P holds), batches of 4, each batch's output copied to the host
    and accumulated there.  forward: the BS-Roformer oracle's, or the Mel-Band Roformer oracle's"""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    dev = torch.device("cuda")

    def net(a):
        a = a.to(dev)
        with torch.autocast("cuda", enabled=autocast), sdpa_kernel([SDPBackend.MATH, SDPBackend.EFFICIENT_ATTENTION]):
            return forward(P, cfg, a.half() if half else a).float().cpu()

    return BR.demix_track(net, mix)["vocals"]


MEL_FAMILIES = (("gemm", ("evk_gconv_fwd", "evk_linear_h16")), ("attention", ("evk_rope_attn_fwd", "evk_rope_attn_fwd_h16")),
                ("norms", ("evk_row_norm",)),
                ("band_input", ("evk_band_input",)), ("melband_mask_avg", ("evk_melband_mask_avg",)),
                ("stft_istft", ("evk_stft_fwd", "evk_istft")))


def roformer_main(a):
    assert torch.cuda.is_available(), "needs a GPU"
    from easevoice_trainer_b200 import bs_roformer, lib, mel_band_roformer, ops
    lib.init().evk_set_precise(0)
    if a.net == "melroformer":
        cfg, families, forward = dict(MR.DEFAULT), MEL_FAMILIES, MR.forward
        P = MR.init_params(MR.param_spec(cfg), 181)
        model = mel_band_roformer.MelBandRoformer(**cfg).to("cuda").load_state_dict(P)
    else:
        cfg, families, forward = dict(BR.SHIPPED), FAMILIES, BR.forward
        P = BR.init_params(BR.param_spec(cfg), 81)
        model = bs_roformer.BSRoformer(**cfg).to("cuda").load_state_dict(P)
    mix = BR.make_audio(7, (2, 7938000))
    res = dict(gpu=gpu_info(), net=a.net, samples=mix.shape[1], chunks=-(-mix.shape[1] // BR.CHUNK), max_chunks=a.max_chunks)
    # the fp32 (TF32) arm's results at the top level; a 16-bit arm's under its --precision name.  The arms alternate in the
    # timed calls, so both see the same card state.
    arms = [("float32", None, res)]
    if a.precision != "float32":
        res[a.precision] = {}
        arms.append((a.precision, getattr(torch, a.precision), res[a.precision]))
    outs = {}
    for name, dt, r in arms:
        model.set_compute_type(dt)
        t = time.perf_counter()
        outs[name] = bs_roformer.demix_track(model, mix, "cuda", a.max_chunks)["vocals"]
        r["evk_first_call_s"] = round(time.perf_counter() - t, 3)
        r["evk_s"], r["peak_mem_gib"] = [], 0.0
    for _ in range(a.reps):
        for name, dt, r in arms:
            model.set_compute_type(dt)
            torch.cuda.reset_peak_memory_stats()
            r["evk_s"] += [round(t, 3) for t in timed(lambda: bs_roformer.demix_track(model, mix, "cuda", a.max_chunks), 1)]
            r["peak_mem_gib"] = max(r["peak_mem_gib"], round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    batch = mix[:, :a.max_chunks * BR.CHUNK].reshape(2, a.max_chunks, BR.CHUNK).transpose(0, 1).contiguous().cuda()
    for name, dt, r in arms:
        model.set_compute_type(dt)
        model.forward(batch)
        ops.profile_begin()
        model.forward(batch)
        prof = ops.profile_end()
        tot = sum(v["ms"] for v in prof.values())
        fam = {n: round(sum(v["ms"] for k, v in prof.items() if k.split(":")[0] in keys), 2) for n, keys in families}
        fam["other"] = round(tot - sum(fam.values()), 2)
        r["forward_ms_by_family"] = fam
        r["forward_device_ms"] = round(tot, 2)
        gemm_fl = sum(v["flops"] for k, v in prof.items() if k.split(":")[0] in families[0][1])
        r["chunk_tflop_gemm"] = round(gemm_fl / a.max_chunks / 1e12, 2)
        r["gemm_tflops_in_forward"] = round(gemm_fl / fam["gemm"] / 1e9, 1)
        if a.net == "roformer":
            r["rope_attn"] = rope_attn_rates(ops, dtype=dt)
    model.set_compute_type(None)
    out = outs["float32"]
    if a.precision != "float32":
        res[a.precision]["rel_l2_vs_evk_float32"] = float(np.linalg.norm(outs[a.precision] - out) / np.linalg.norm(out))
    if not a.skip_torch:
        torch.backends.cudnn.allow_tf32 = True
        small = BR.make_audio(8, (2, BR.CHUNK))
        rel = lambda x, r: float(np.linalg.norm(x - r) / np.linalg.norm(r))  # noqa: E731
        # accuracy yardstick: the same algorithm in fp32 with TF32 off (one run, not timed)
        torch.backends.cuda.matmul.allow_tf32 = False
        Pd = {k: v.cuda() for k, v in P.items()}
        exact = torch_roformer_demix(Pd, cfg, mix, False, False, forward)
        res["evk_rel_l2_vs_torch_fp32"] = rel(out, exact)
        if a.precision != "float32":
            res[a.precision]["rel_l2_vs_torch_fp32"] = rel(outs[a.precision], exact)
        torch.backends.cuda.matmul.allow_tf32 = True
        # (name, weights in fp16, chunks in fp16, autocast): the shipped cfg.is_half path, then fp32 with TF32 allowed
        arms = [("torch_fp16", True, True, True), ("torch_tf32", False, False, False)]
        while arms:
            name, wh, ch, ac = arms.pop(0)
            Pd = {k: (v.half() if wh else v).cuda() for k, v in P.items()}
            try:
                torch_roformer_demix(Pd, cfg, small, ch, ac, forward)                  # warm-up
            except RuntimeError as e:
                if name != "torch_fp16":
                    raise
                # the is_half configuration as written does not run: record why, then autocast with fp32 weights
                res["torch_fp16_error"] = f"{type(e).__name__}: {str(e)[:300]}"
                arms.insert(0, ("torch_autocast_fp32_weights", False, False, True))
                continue
            ts = timed(lambda: torch_roformer_demix(Pd, cfg, mix, ch, ac, forward), a.reps)
            res[name + "_s"] = [round(t, 3) for t in ts]
            ref = torch_roformer_demix(Pd, cfg, mix, ch, ac, forward)
            res[name + "_rel_l2_vs_evk"] = rel(ref, out)
            res[name + "_rel_l2_vs_torch_fp32"] = rel(ref, exact)
            if a.precision != "float32":
                res[a.precision][name + "_rel_l2_vs_evk"] = rel(ref, outs[a.precision])
            del Pd
            torch.cuda.empty_cache()
    print(json.dumps(res))


WAVE_FAMILIES = ("evk_vr_band_stft", "evk_vr_mag_norm", "evk_resample_poly", "evk_vr_assemble", "evk_istft")


def mdx_conv_flops(cfg, B):
    """-> {family: FLOPs} of one forward of B chunks, computed from the layer shapes (2 per multiply-add)"""
    a, m = cfg["audio"], cfg["model"]
    T, F_ = a["chunk_size"] // a["hop_length"] + 1, a["dim_f"] // m["num_subbands"]
    k, S, n, l, c, g, bn = (m["num_subbands"], a["num_channels"], m["num_scales"], m["num_blocks_per_scale"],
                            m["num_channels"], m["growth"], m["bottleneck_factor"])
    nt = 1 if cfg["training"]["target_instrument"] else len(cfg["training"]["instruments"])
    D = 2 * S * k
    fl = dict(conv3x3=0.0, conv2x2=0.0, conv1x1=0.0, tdf=0.0)

    def block(in_c, c, h, w):
        for _ in range(l):
            fl["conv3x3"] += 2 * B * h * w * 9 * (in_c * c + c * c)
            fl["conv1x1"] += 2 * B * h * w * in_c * c
            fl["tdf"] += 2 * 2 * B * h * c * w * (w // bn)
            in_c = c

    h, w = T, F_
    fl["conv1x1"] += 2 * B * h * w * D * c + 2 * B * h * w * ((c + D) * c + c * nt * D)
    for _ in range(n):
        block(c, c, h, w)
        fl["conv2x2"] += 2 * B * (h // 2) * (w // 2) * 4 * c * (c + g)
        h, w, c = h // 2, w // 2, c + g
    block(c, c, h, w)
    for _ in range(n):
        fl["conv2x2"] += 2 * B * h * w * 4 * c * (c - g)
        h, w, c = h * 2, w * 2, c - g
        block(2 * c, c, h, w)
    return fl


MDX_FAMILIES = (("conv3x3_1x1", ("evk_conv2d_fwd",)), ("conv2x2_down", ("evk_conv2d_fwd_k2",)),
                ("conv2x2_up", ("evk_convt2x2_fwd",)), ("tdf", ("evk_mdx_tdf",)), ("instnorm", ("evk_instnorm_plane",)),
                ("stft_istft", ("evk_stft_fwd", "evk_istft")))


def mdx_main(a):
    """--net mdx23c: MDX23C at the 8K-FFT InstVoc configuration"""
    assert torch.cuda.is_available(), "needs a GPU"
    from easevoice_trainer_b200 import bs_roformer, lib, mdx23c, ops
    lib.init().evk_set_precise(0)
    cfg = MX.config({})
    P = MX.init_params(MX.param_spec(cfg), 321)
    model = mdx23c.MDX23C(cfg).to("cuda").load_state_dict(P)
    c = cfg["audio"]["chunk_size"]
    mix = BR.make_audio(7, (2, 7938000))
    res = dict(gpu=gpu_info(), net=a.net, samples=mix.shape[1], chunks=-(-mix.shape[1] // c), max_chunks=a.max_chunks)
    t = time.perf_counter()
    out = bs_roformer.demix_track(model, mix, "cuda", a.max_chunks)
    res["evk_first_call_s"] = round(time.perf_counter() - t, 3)
    torch.cuda.reset_peak_memory_stats()
    ts = timed(lambda: bs_roformer.demix_track(model, mix, "cuda", a.max_chunks), a.reps)
    res["evk_s"] = [round(t, 3) for t in ts]
    res["peak_mem_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    batch = mix[:, :a.max_chunks * c].reshape(2, a.max_chunks, c).transpose(0, 1).contiguous().cuda()
    model.forward(batch)
    ops.PROF_SHAPES = True                 # conv2d's profile keys then carry the kernel size, which splits 2x2 from 3x3 / 1x1
    ops.profile_begin()
    model.forward(batch)
    prof = ops.profile_end()
    ops.PROF_SHAPES = False
    agg = {}
    for key, v in prof.items():
        name = key.split("|")[0].split(":")[0]
        if name == "evk_conv2d_fwd" and key.endswith("|k2"):
            name = "evk_conv2d_fwd_k2"
        e = agg.setdefault(name, dict(ms=0.0, flops=0.0))
        e["ms"] += v["ms"]
        e["flops"] += v["flops"]
    tot = sum(v["ms"] for v in agg.values())
    fam = {name: round(sum(v["ms"] for k, v in agg.items() if k in keys), 2) for name, keys in MDX_FAMILIES}
    fam["other"] = round(tot - sum(fam.values()), 2)
    res["forward_ms_by_family"] = fam
    res["forward_device_ms"] = round(tot, 2)
    fl = mdx_conv_flops(cfg, a.max_chunks)
    res["chunk_tflop_by_family"] = {k: round(v / a.max_chunks / 1e12, 3) for k, v in fl.items()}
    conv_ms = fam["conv3x3_1x1"] + fam["conv2x2_down"] + fam["conv2x2_up"]
    res["conv_tflops_in_forward"] = round((fl["conv3x3"] + fl["conv1x1"] + fl["conv2x2"]) / conv_ms / 1e9, 1)
    res["tdf_tflops_in_forward"] = round(fl["tdf"] / fam["tdf"] / 1e9, 1)
    if not a.skip_torch:
        rel = lambda x, r: float(np.linalg.norm(x - r) / np.linalg.norm(r))  # noqa: E731
        small = BR.make_audio(8, (2, c))
        ev = np.stack([out["vocals"], out["other"]])
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cuda.matmul.allow_tf32 = True
        arms = [("torch_fp16", True, True, True), ("torch_tf32", False, False, False)]
        while arms:
            name, wh, ch, ac = arms.pop(0)
            Pd = {k: (v.half() if wh else v).cuda() for k, v in P.items()}

            def net(x):
                x = x.cuda()
                with torch.no_grad(), torch.autocast("cuda", enabled=ac):
                    return MX.forward(Pd, cfg, x.half() if ch else x).float().cpu()
            try:
                MX.demix_track(net, small, c)                                      # warm-up
            except RuntimeError as e:
                if name != "torch_fp16":
                    raise
                res["torch_fp16_error"] = f"{type(e).__name__}: {str(e)[:300]}"
                arms.insert(0, ("torch_autocast_fp32_weights", False, False, True))
                continue
            ts = timed(lambda: MX.demix_track(net, mix, c), a.reps)
            res[name + "_s"] = [round(t, 3) for t in ts]
            ref = MX.demix_track(net, mix, c)
            res[name + "_rel_l2_vs_evk"] = rel(np.stack([ref["vocals"], ref["other"]]), ev)
            del Pd
            torch.cuda.empty_cache()
    print(json.dumps(res))


def wave_main(a):
    """--wave: uvr5.separate_wave against the reference's host front / back end around uvr5.inference"""
    assert torch.cuda.is_available(), "needs a GPU"
    from easevoice_trainer_b200 import lib, ops, uvr5
    from oracle import uvr5_wave_oracle as W
    lib.init().evk_set_precise(0)
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_wave.pt"), weights_only=False)
    if a.net == "vr":
        param = gold["vr"]["param"]
        net = uvr5.get_nets_model(1344).to("cuda").load_state_dict(O.init_params(O.param_spec(61968), 31))
    else:
        param = gold["echo"]["param"]
        nout = 48 if a.net == "deecho" else 64
        net = uvr5.CascadedNet(1344, nout).to("cuda").load_state_dict(E.init_params(E.param_spec(1344, nout), 51))
    mix = W.make_clip(7, 180.0, extra=0)
    assert mix.shape == (2, 7938000)
    res = dict(gpu=gpu_info(), net=a.net, wave=True, samples=mix.shape[1], tta=bool(a.tta), max_windows=a.max_windows)
    run = lambda: uvr5.separate_wave(mix, net, param, 10, bool(a.tta), max_windows=a.max_windows)  # noqa: E731
    t = time.perf_counter()
    acc, _ = run()
    res["evk_first_call_s"] = round(time.perf_counter() - t, 3)
    res["l"] = acc.shape[0] // 480 + 1
    torch.cuda.reset_peak_memory_stats()
    res["evk_separate_wave_s"] = [round(t, 3) for t in timed(run, a.reps)]
    res["peak_mem_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    ops.profile_begin()
    run()
    prof = ops.profile_end()
    new = sum(v["ms"] for k, v in prof.items() if k.split(":")[0] in WAVE_FAMILIES)
    tot = sum(v["ms"] for v in prof.values())
    res["device_ms_front_back_kernels"] = round(new, 1)
    res["device_ms_all_library_calls"] = round(tot, 1)
    res["device_ms_by_new_kernel"] = {k: round(v["ms"], 2) for k, v in prof.items() if k.split(":")[0] in WAVE_FAMILIES}
    if not a.skip_torch:
        agg = {"value": 0.1, "split_bin": param["band"][1]["crop_stop"], "aggr_correction": None}
        data = {"window_size": 512, "tta": bool(a.tta)}
        split = dict(front=[], net=[], back=[])
        for _ in range(a.reps):
            t0 = time.perf_counter()
            x_spec_m, ihe_h, ihe = W.front_end(mix, param)
            t1 = time.perf_counter()
            pred, _, phase = uvr5.inference(x_spec_m, "cuda", net, agg, data, a.max_windows)
            t2 = time.perf_counter()
            W.back_end(x_spec_m, pred, phase, param, ihe_h, ihe)
            t3 = time.perf_counter()
            for k, v in zip(split, (t1 - t0, t2 - t1, t3 - t2)):
                split[k].append(round(v, 3))
        res["host_path_s"] = split
    print(json.dumps(res))


def h16_main(a):
    """--precision float16 | bfloat16 with --net vr / deecho / dereverb / mdx23c (and --wave): the fp32 and 16-bit arms of
    the library alternating in one process"""
    assert torch.cuda.is_available(), "needs a GPU"
    from easevoice_trainer_b200 import bs_roformer, lib, mdx23c, ops, uvr5
    from oracle import uvr5_wave_oracle as W
    lib.init().evk_set_precise(0)
    dt = getattr(torch, a.precision)
    agg = {"value": 0.1, "split_bin": 85, "aggr_correction": None}
    if a.net == "mdx23c":
        cfg = MX.config({})
        net = mdx23c.MDX23C(cfg).to("cuda").load_state_dict(MX.init_params(MX.param_spec(cfg), 321))
        mix = BR.make_audio(7, (2, 7938000))
        c = cfg["audio"]["chunk_size"]
        run = lambda: np.stack(list(bs_roformer.demix_track(net, mix, "cuda", a.max_chunks).values()))  # noqa: E731
        batch = mix[:, :a.max_chunks * c].reshape(2, a.max_chunks, c).transpose(0, 1).contiguous().cuda()
        forward = lambda: net.forward(batch)                                                        # noqa: E731
    else:
        if a.net == "vr":
            net = uvr5.get_nets_model(1344).to("cuda").load_state_dict(O.init_params(O.param_spec(61968), 31))
        else:
            nout = 48 if a.net == "deecho" else 64
            net = uvr5.CascadedNet(1344, nout).to("cuda").load_state_dict(E.init_params(E.param_spec(1344, nout), 51))
        if a.wave:
            gold = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_wave.pt"), weights_only=False)
            param = gold["vr" if a.net == "vr" else "echo"]["param"]
            mix = W.make_clip(7, 180.0, extra=0)
            run = lambda: np.stack(uvr5.separate_wave(mix, net, param, 10, bool(a.tta), max_windows=a.max_windows))  # noqa: E731
        else:
            spec = O.make_spec(7, 673, a.frames)
            data = {"window_size": 512, "tta": bool(a.tta)}
            run = lambda: uvr5.inference(spec, "cuda", net, agg, data, a.max_windows)[0]          # noqa: E731
        wins = torch.rand(a.max_windows, 2, 673, 512, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
        forward = lambda: net.predict(wins, agg)                                                  # noqa: E731
    res = dict(gpu=gpu_info(), net=a.net, wave=bool(a.wave), tta=bool(a.tta), precision=a.precision,
               max_windows=a.max_windows, max_chunks=a.max_chunks)
    arms = (("float32", None), (a.precision, dt))
    outs, times, peak = {}, {n: [] for n, _ in arms}, {}
    for name, ct in arms:                                 # first calls: packing, allocator growth, module loads
        net.set_compute_type(ct)
        outs[name] = run()
    for _ in range(a.reps):
        for name, ct in arms:
            net.set_compute_type(ct)
            torch.cuda.reset_peak_memory_stats()
            times[name] += timed(run, 1)
            peak[name] = max(peak.get(name, 0.0), torch.cuda.max_memory_allocated() / 2 ** 30)
    for name, ct in arms:
        net.set_compute_type(ct)
        forward()
        ops.profile_begin()
        forward()
        prof = ops.profile_end()
        conv = [v for k, v in prof.items() if k.startswith("evk_conv2d_fwd")]
        conv_ms, conv_fl = sum(v["ms"] for v in conv), sum(v["flops"] for v in conv)
        tot = sum(v["ms"] for v in prof.values())
        res[name] = dict(call_s=[round(t, 3) for t in times[name]], peak_mem_gib=round(peak[name], 2),
                         forward_device_ms=round(tot, 2), conv_ms=round(conv_ms, 2), other_ms=round(tot - conv_ms, 2),
                         conv_tflops=round(conv_fl / conv_ms / 1e9, 1),
                         other_ms_by_family={k: round(v["ms"], 2) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])
                                             if not k.startswith("evk_conv2d_fwd")})
    ref, got = outs["float32"].astype(np.float64), outs[a.precision].astype(np.float64)
    res[a.precision]["finite"] = bool(np.isfinite(got).all())
    res[a.precision]["rel_l2_vs_float32"] = float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
    net.set_compute_type(None)
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", choices=("vr", "deecho", "dereverb", "roformer", "melroformer", "mdx23c"), default="vr")
    ap.add_argument("--max-chunks", type=int, default=4)
    ap.add_argument("--frames", type=int, default=16538)
    ap.add_argument("--tta", type=int, default=0)
    ap.add_argument("--max-windows", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-torch", action="store_true")
    ap.add_argument("--precision", choices=("float32", "float16", "bfloat16"), default="float32",
                    help="also run this 16-bit compute type, alternating with the fp32 arm")
    ap.add_argument("--wave", action="store_true")
    a = ap.parse_args()
    if a.precision != "float32" and a.net not in ("roformer", "melroformer"):
        return h16_main(a)
    if a.wave:
        return wave_main(a)
    if a.net in ("roformer", "melroformer"):
        return roformer_main(a)
    if a.net == "mdx23c":
        return mdx_main(a)
    if a.net != "vr":
        return echo_main(a)
    assert torch.cuda.is_available(), "needs a GPU"
    from easevoice_trainer_b200 import lib, ops, uvr5
    lib.init().evk_set_precise(0)
    P = O.init_params(O.param_spec(61968), 31)
    net = uvr5.get_nets_model(1344).to("cuda").load_state_dict(P)
    spec = O.make_spec(7, 673, a.frames)
    agg = {"value": 0.1, "split_bin": 85, "aggr_correction": None}
    data = {"window_size": 512, "tta": bool(a.tta)}
    n_win = int(np.ceil(a.frames / 256)) * (2 if a.tta else 1) + (1 if a.tta else 0)
    res = dict(gpu=gpu_info(), frames=a.frames, tta=bool(a.tta), windows=n_win, max_windows=a.max_windows)

    t = time.perf_counter()
    uvr5.inference(spec, "cuda", net, agg, data, a.max_windows)      # first call: the allocator grows to the batch's size
    res["evk_first_call_s"] = round(time.perf_counter() - t, 3)
    ops.profile_begin()
    net.predict(torch.rand(a.max_windows, 2, 673, 512, device="cuda"), agg)
    prof = ops.profile_end()
    conv = prof.get("evk_conv2d_fwd", dict(ms=0.0, flops=0.0))
    res["window_gflop"] = round(conv["flops"] / a.max_windows / 1e9, 1)
    res["conv2d_share_of_predict_ms"] = round(conv["ms"] / sum(v["ms"] for v in prof.values()), 3)
    res["conv2d_tflops_in_predict"] = round(conv["flops"] / conv["ms"] / 1e9, 1)
    ts = timed(lambda: uvr5.inference(spec, "cuda", net, agg, data, a.max_windows), a.reps)
    res["evk_s"] = [round(t, 3) for t in ts]
    res["evk_tflops_end_to_end"] = round(res["window_gflop"] * n_win / min(ts) / 1e3, 1)
    t = time.perf_counter()
    np.exp(1.0j * np.angle(spec))
    res["host_phase_s"] = round(time.perf_counter() - t, 3)          # overlapped with the net inside inference()
    wins = torch.rand(n_win, 2, 673, 512, device="cuda")
    res["evk_net_only_s"] = [round(t, 3) for t in timed(
        lambda: [net.predict(wins[i:i + a.max_windows], agg) for i in range(0, n_win, a.max_windows)], a.reps)]
    del wins
    res["decoder_conv2d"] = decoder_rates(ops, a.max_windows)
    pred = uvr5.inference(spec, "cuda", net, agg, data, a.max_windows)[0]

    if not a.skip_torch:
        torch.backends.cudnn.benchmark = True
        for name, half in (("torch_fp16", True), ("torch_tf32", False)):
            torch.backends.cudnn.allow_tf32 = True
            torch_inference(P, O.make_spec(1, 673, 600), agg, data, half)             # warm-up (cuDNN algorithm choice)
            ts = timed(lambda: torch_inference(P, spec, agg, data, half), a.reps)
            res[name + "_s"] = [round(t, 3) for t in ts]
            ref = torch_inference(P, spec, agg, data, half)[0]
            res[name + "_rel_l2_vs_evk"] = float(np.linalg.norm(ref - pred) / np.linalg.norm(ref))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
