#!/usr/bin/env python
"""Benchmark of the stage-2 (SoVITS + HiFi-GAN) train step -- BASELINE.json's metric.

  python bench.py --gpus N --steps K --warmup W            # this repo's sm_90a path (N>1: launched by torchrun)
  python bench.py --impl reference --steps K --warmup W    # the reference's algorithm on the host CPU cores (oracle port)
  python bench.py ... --dump-outputs DIR                   # also write the last timed step's results as DIR/<name>.npy

One "step" = everything in the reference's src/train/sovits.py:438-525 for one batch of 16 x 10 s utterances:
G forward, mel features + slicing, D forward/backward/AdamW, D forward again, G backward/AdamW.
`value` is device-timed with the batch resident in HBM; `e2e` adds, every step, the pinned-host -> device copy of the
step's inputs (wav, ssl features, phonemes, lengths), the on-GPU |X| feature extraction the reference does in CPU
DataLoader workers, and a device -> host read of the step's losses.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "s2 SoVITS+HiFiGAN train-step audio-seconds/sec"
UNIT = "audio-s/s"
B_PER_GPU, UTT_SECONDS, TEXT_LEN, HOP = 16, 10.0, 120, 640


def frames_for(sr_label):
    T = int(UTT_SECONDS * sr_label) // HOP
    return 2 * (T // 2 + 1)                    # TextAudioSpeakerCollate pads to 2*(Tmax//2+1) (data_utils.py:185-188)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d["bf16_tflops"], d.get("bf16_tflops_sustained", d["bf16_tflops"]), "measured"
    return 3350.0, 989.0, 989.0, "H100 SXM data sheet (dense; not a measured rate)"


class ClockSampler(threading.Thread):
    """nvidia-smi clocks/throttle reasons every 200 ms during the timed region (read-only queries)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.proc = index, [], None

    def run(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "200",
                                          "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                self.rows.append([c.strip() for c in line.split(",")])
        except Exception:
            pass

    def stop(self):
        if self.proc:
            self.proc.terminate()
        time.sleep(0.05)
        sm = sorted(int(float(r[1])) for r in self.rows if len(r) >= 9 and r[1].replace(".", "").isdigit())
        reasons = set()
        for r in self.rows:
            if len(r) >= 9:
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
        mx = max((int(float(r[2])) for r in self.rows if len(r) >= 9 and r[2].replace(".", "").isdigit()), default=None)
        return dict(sm_mhz=(sm[len(sm) // 2] if sm else None), sm_max_mhz=mx, reasons=sorted(reasons), samples=len(sm))


# --------------------------------------------------------------------------------------------------
def cpu_threads():
    """Threads for the CPU arm: torch's intra-op pool stops scaling (and then degrades badly) on these small conv
    shapes well before 128 threads -- measured 550 s/step with 128 threads vs ~7 s with 8 -- so use at most 16."""
    return max(1, min(os.cpu_count() or 1, 16))


def _oracle_leaves(s2_oracle, seed_g=1234, seed_d=4321, dev="cpu"):
    PG = {k: v.to(dev) for k, v in s2_oracle.init_params(s2_oracle.generator_param_spec(), seed_g).items()}
    PD = {k: v.to(dev) for k, v in s2_oracle.init_params(s2_oracle.discriminator_param_spec(), seed_d).items()}
    for k, v in PG.items():
        if k not in s2_oracle.GEN_BUFFERS:
            v.requires_grad_(True)
    for v in PD.values():
        v.requires_grad_(True)
    gp = [v for k, v in PG.items() if k not in s2_oracle.GEN_BUFFERS and not k.startswith("ssl_proj.")]
    return PG, PD, gp


def cpu_reference_step(Bc, T, threads, steps, warmup, budget_s=None):
    """The reference's algorithm (oracle port of sovits.py:459-525, torch fp32, CPU) on `Bc` utterances per step:
    forward, D backward + AdamW, G backward + AdamW -- the whole optimisation step, like the GPU arm.
    -> (mean seconds per timed step, timed steps actually run).  budget_s bounds the wall time of the timed region."""
    import torch
    from oracle import s2_oracle, mel_oracle
    torch.set_num_threads(threads)
    PG, PD, gp = _oracle_leaves(s2_oracle)
    opt_d = torch.optim.AdamW(list(PD.values()), 1e-4, betas=(0.8, 0.99), eps=1e-9)
    opt_g = torch.optim.AdamW(gp, 1e-4, betas=(0.8, 0.99), eps=1e-9)
    wav, ssl, text, spec_len, text_len = s2_oracle.synthetic_batch(Bc, T, TEXT_LEN, 1234)
    spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, HOP, 2048)
    g = torch.Generator().manual_seed(1)
    times = []
    t_begin = time.perf_counter()
    for it in range(warmup + steps):
        noise = torch.randn(Bc, 192, T, generator=g)
        ids = (torch.rand(Bc, generator=g) * (spec_len - 32 + 1)).long()
        t0 = time.perf_counter()
        o = s2_oracle.s2_losses(PG, PD, (ssl, spec, spec_len, wav, text, text_len), noise, ids)
        opt_d.zero_grad(set_to_none=True)
        for p_, g_ in zip(PD.values(), torch.autograd.grad(o["loss_disc"], list(PD.values()), retain_graph=True)):
            p_.grad = g_
        opt_d.step()
        opt_g.zero_grad(set_to_none=True)
        for p_, g_ in zip(gp, torch.autograd.grad(o["loss_gen_all"], gp)):
            p_.grad = g_
        opt_g.step()
        dt = time.perf_counter() - t0
        if it >= warmup:
            times.append(dt)
            if budget_s is not None and time.perf_counter() - t_begin + dt > budget_s:
                break
    return sum(times) / len(times), len(times)


def torch_gpu_port_step(dev, T, amp, steps=5):
    """The reference's algorithm through STOCK PyTorch kernels (cuDNN / cuBLAS / cuFFT / ATen) on the same GPU, B = 16,
    whole optimisation step (two torch.optim.AdamW updates): the oracle port moved to the GPU.
      amp=False: fp32 storage, TF32 allowed exactly as the reference sets it (sovits.py:172-176);
      amp=True : the reference's AS-SHIPPED regime (configs/s2.json fp16_run: true): torch.autocast(float16) around the
                 networks, losses in fp32, GradScaler on both optimizers (sovits.py:378,459-525).
    The reference package itself is not installed next to this one, so its
    restated algorithm stands in for it; this is the 'reference 1-GPU PyTorch step' of BASELINE.json's >= 10x target."""
    import torch
    from oracle import s2_oracle, mel_oracle
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    PG, PD, gp = _oracle_leaves(s2_oracle, dev=dev)
    opt_d = torch.optim.AdamW(list(PD.values()), 1e-4, betas=(0.8, 0.99), eps=1e-9)
    opt_g = torch.optim.AdamW(gp, 1e-4, betas=(0.8, 0.99), eps=1e-9)
    scaler = torch.amp.GradScaler("cuda", enabled=amp)
    wav, ssl, text, spec_len, text_len = [t.to(dev) for t in s2_oracle.synthetic_batch(B_PER_GPU, T, TEXT_LEN, 1234)]
    spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, HOP, 2048)
    g = torch.Generator(device=dev).manual_seed(1)
    data, train = s2_oracle.S2_DATA, s2_oracle.S2_TRAIN
    seg = train["segment_size"] // data["hop_length"]
    margs = (data["filter_length"], data["n_mel_channels"], data["sampling_rate"], data["mel_fmin"], data["mel_fmax"])
    ms = []
    for it in range(steps + 3):
        noise = torch.randn(B_PER_GPU, 192, T, generator=g, device=dev)
        ids = (torch.rand(B_PER_GPU, generator=g, device=dev) * (spec_len - 32 + 1)).long()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            out = s2_oracle.synthesizer_forward(PG, ssl, spec, spec_len, text, text_len, noise, ids, s2_oracle.S2_MODEL, seg)
            y_hat = out["y_hat"]
            mel = mel_oracle.spec_to_mel(spec, *margs)
            y_mel = s2_oracle.slice_segments(mel, ids, seg)
            y_hat_mel = mel_oracle.mel_spectrogram(y_hat.squeeze(1).float(), data["filter_length"], data["n_mel_channels"],
                                                   data["sampling_rate"], data["hop_length"], data["win_length"], data["mel_fmin"], data["mel_fmax"])
            y = s2_oracle.slice_segments(wav, ids * data["hop_length"], train["segment_size"])
            rs, gs, _, _ = s2_oracle.mpd(PD, y, y_hat.detach())
            with torch.autocast("cuda", enabled=False):
                loss_disc = s2_oracle.discriminator_loss([t.float() for t in rs], [t.float() for t in gs])
        opt_d.zero_grad(set_to_none=True)
        scaler.scale(loss_disc).backward()
        scaler.unscale_(opt_d)
        scaler.step(opt_d)
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            rs, gs, frs, fgs = s2_oracle.mpd(PD, y, y_hat)
            with torch.autocast("cuda", enabled=False):
                loss_mel = torch.nn.functional.l1_loss(y_mel.float(), y_hat_mel.float()) * train["c_mel"]
                loss_kl = s2_oracle.kl_loss(out["z_p"].float(), out["logs_q"].float(), out["m_p"].float(), out["logs_p"].float(), out["y_mask"]) * train["c_kl"]
                loss_fm = s2_oracle.feature_loss([[t.float() for t in f] for f in frs], [[t.float() for t in f] for f in fgs])
                loss_gen = s2_oracle.generator_loss([t.float() for t in gs])
                total = loss_gen + loss_fm + loss_mel + loss_kl
        opt_g.zero_grad(set_to_none=True)
        for p_ in PD.values():
            p_.grad = None
        scaler.scale(total).backward()
        scaler.unscale_(opt_g)
        scaler.step(opt_g)
        scaler.update()
        e1.record()
        torch.cuda.synchronize()
        if it >= 3:
            ms.append(e0.elapsed_time(e1))
    ms.sort()
    return ms[len(ms) // 2], float(total)


def run_reference(args):
    """`--impl reference`: the reference's CPU path for the same workload / config / metric.  The reference package cannot be
    installed next to this one, so the arm runs its restated algorithm (oracle port, kind "port") on
    the host's CPU cores at the FULL benchmark batch (16 x 10 s), whole optimisation step.  Rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    threads = cpu_threads()
    T = frames_for(args.sr_label)
    Bc = args.cpu_batch if args.cpu_batch > 0 else B_PER_GPU
    warm = min(args.warmup, 1)
    sec, n_timed = cpu_reference_step(Bc, T, threads, args.steps, warm, budget_s=args.cpu_budget)
    val = Bc * UTT_SECONDS / sec
    sample = (f"oracle port of sovits.py:459-525 (fwd, D bwd + AdamW, G bwd + AdamW; fp32), B={Bc} x {UTT_SECONDS:.0f} s (T={T}), {threads} threads, "
              f"{warm} warm-up + {n_timed} timed steps (wall-time budget {args.cpu_budget:.0f} s)")
    line = dict(metric=METRIC, value=val, unit=UNIT, n_gpus=args.gpus, steps=n_timed, warmup=warm,
                ms_per_step=sec * 1e3, higher_is_better=True, scaling="weak", vs_baseline=None, dtype="f32", data="synthetic",
                impl="reference", config=workload_config(args.sr_label, max(args.gpus, 1)),
                cpu_baseline=dict(value=val, unit=UNIT, cores=threads, kind="port", sample=sample),
                e2e=dict(value=val, unit=UNIT, h2d_bytes_per_step=0, d2h_bytes_per_step=0))
    emit(line)
    return 0


def workload_config(sr_label, world):
    """identical for both arms (the driver compares them): BASELINE config 3 / 4."""
    T = frames_for(sr_label)
    return dict(workload=f"s2_step_B{B_PER_GPU}x{UTT_SECONDS:.0f}s_sr{sr_label}_T{T}", global_batch=world * B_PER_GPU, frames=T,
                segment=20480, text_len=TEXT_LEN, parallelism=f"dp{world}", weights="random-init seed 1234",
                l2="params+optimizer state+activations touched per step (>2 GB) far exceed the 50 MB L2 of an H100; no explicit flush")


# --------------------------------------------------------------------------------------------------
def graph_time(fn):
    """Device time (ms) of `fn`'s launches with the host taken out of the loop: capture once, time a graph replay."""
    import torch
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernel_table(ops, dev):
    """Heaviest conv layers of the step (Appendix A of SURVEY.md), forward launch of each timed in isolation.
    count = how many times a launch of that shape/flop count runs per step (fwd + dgrad of G and of the 2B-batched D)."""
    import torch
    B = B_PER_GPU
    rows = []
    #        name, batch, T, C, N, k, dil, P, stride, launches/step
    layers = [("dec stage1 resblock k11 128ch", B, 2560, 128, 128, 11, 1, 1, 1, 12), ("dec stage1 resblock k7 128ch", B, 2560, 128, 128, 7, 1, 1, 1, 12),
              ("dec stage0 resblock k11 256ch", B, 320, 256, 256, 11, 1, 1, 1, 12), ("dec stage2 resblock k11 64ch", B, 5120, 64, 64, 11, 1, 1, 1, 12),
              ("dec stage3 resblock k11 32ch", B, 10240, 32, 32, 11, 1, 1, 1, 12), ("dec stage4 resblock k11 16ch", B, 20480, 16, 16, 11, 1, 1, 1, 12),
              ("discP 1024->1024 k5 p=2", 2 * B, 127, 1024, 1024, 5, 1, 2, 1, 4), ("discP 512->1024 k5 s3 p=2", 2 * B, 380, 512, 1024, 5, 1, 2, 3, 4),
              ("discS 1024->1024 k5", 2 * B, 80, 1024, 1024, 5, 1, 1, 1, 4), ("enc_q WN in_layer 192->384 k5", B, 346, 192, 384, 5, 1, 1, 1, 32),
              ("enc_p FFN 192->768 k3", B, 346, 192, 768, 3, 1, 1, 1, 12)]
    for name, b, T, C, N, k, dil, P, stride, count in layers:
        nset = 6
        xs = [torch.randn(b, T * P, C, device=dev) for _ in range(nset)]
        v = torch.randn(N, C, k, device=dev) * 0.02
        w = ops.pack_weight(v, None)
        bias = torch.zeros(N, device=dev)
        pad = (k * dil - dil) // 2
        def burst():
            for _ in range(4):
                for x in xs:
                    yy = ops.conv(x, w, bias, stride=stride, pad=pad, dil=dil, P=P)
            return yy
        with torch.no_grad():
            y = burst()
            ms = graph_time(burst) / (4 * nset)
        J = y.shape[1]
        flops = 2.0 * b * J * N * C * k
        rows.append(dict(layer=name, ms=ms, flops=flops, tflops=flops / (ms * 1e-3) / 1e12, count=count))
        del xs
    return rows


def dump_outputs(dirpath, arrays):
    """--dump-outputs: one DIR/<name>.npy per array (float32 / float64 only), so that two builds run with the same arguments
    can be compared output for output."""
    import numpy as np
    os.makedirs(dirpath, exist_ok=True)
    total = 0
    for name, a in arrays.items():
        a = np.ascontiguousarray(a)
        assert a.dtype in (np.float32, np.float64), (name, a.dtype)
        total += a.nbytes
        np.save(os.path.join(dirpath, name + ".npy"), a)
    assert total <= 64 * 2**20, total


def param_sample(params, n=1 << 20, seed=0):
    """A fixed, seeded sample of n elements of the concatenated parameters (all of them when there are fewer)."""
    import torch
    flat = torch.cat([p_.detach().reshape(-1).float() for p_ in params])
    if flat.numel() <= n:
        return flat.cpu().numpy()
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(seed))[:n].sort().values
    return flat[idx.to(flat.device)].cpu().numpy()


def trace(msg):
    if os.environ.get("EVK_BENCH_TRACE"):
        print(f"[bench rank {os.environ.get('RANK', '0')} t={time.time() % 1000:.1f}] {msg}", file=sys.stderr, flush=True)


def run_ours(args):
    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from easevoice_trainer_b200 import lib, ops, models
    from easevoice_trainer_b200.train import s2_step
    from easevoice_trainer_b200 import configs
    lib.init()
    trace("lib + process group up")
    if args.config == 5:
        if rank == 0:
            emit(dict(metric="HiFi-GAN generator + MPD/MSD + MR-STFT loss step (BASELINE config 5)", **config5_section(args, dev)))
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return 0
    if args.only_gpt:
        out = gpt_section(args, dev, rank, world)
        if rank == 0:
            emit(out)
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return 0
    hps = configs.load_s2_config()
    torch.manual_seed(hps["train"]["seed"])
    net_g = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                                  n_speakers=hps["data"]["n_speakers"], **hps["model"]).to(dev).train()
    net_d = models.MultiPeriodDiscriminator(hps["model"]["use_spectral_norm"]).to(dev).train()
    st = s2_step.S2Step(net_g, net_d, hps["train"], hps["data"], world_size=world)
    ops.manual_seed(hps["train"]["seed"] + rank)
    T = frames_for(args.sr_label)
    host = s2_step.synthetic_batch(B_PER_GPU, T, TEXT_LEN, dev, seed=1234 + rank)
    host = {k: v.pin_memory() for k, v in host.items()}
    h2d = sum(v.numel() * v.element_size() for v in host.values())

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms) / steps

    batch = s2_step.to_device_batch(host, dev, st.bank)
    trace("batch on device")
    last = {}

    run = st.step if args.no_graph else st.graph_step

    def step_resident():
        last.update(run(batch))

    def step_e2e():
        b = s2_step.to_device_batch(host, dev, st.bank)
        out = run(b)
        last["host"] = torch.stack([out["loss_gen_all"], out["loss_disc"]]).cpu()     # D2H read of the step's losses

    l0 = ops.launches()
    st.step(batch)                                   # one eager step: counts the library launches a step consists of
    launches = ops.launches() - l0
    torch.cuda.synchronize()
    trace("eager step done")
    for _ in range(args.warmup):
        step_resident()
        trace("warm-up step done")
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
        time.sleep(0.3)
    ms = timed(step_resident, args.steps)
    trace(f"timed region done {ms:.1f} ms")
    clocks = sampler.stop() if sampler else None
    if args.dump_outputs and rank == 0:
        # the last timed step's losses and the parameters it left behind (seeded sample of each network)
        import numpy as np
        arrays = {f"loss_{k}": np.asarray([float(v)], dtype=np.float64) for k, v in last.items() if k != "host"}
        arrays["net_g_params_sample"] = param_sample(net_g.parameters())
        arrays["net_d_params_sample"] = param_sample(net_d.parameters())
        dump_outputs(args.dump_outputs, arrays)
    for _ in range(2):
        step_e2e()
    ms_e2e = timed(step_e2e, args.steps)
    audio_s = world * B_PER_GPU * UTT_SECONDS
    losses = {k: float(v) for k, v in last.items() if k != "host"}

    extra = {}
    if rank == 0:
        hbm, tf_burst, tf_sus, src = peaks()
        # ---- dominant kernel, accounted FROM THE STEP: one eager step with a CUDA-event pair around every library call
        #      (ops.profile_begin) and the library's own dispatch accounting telling which kernel family served each
        #      contraction; flops are the analytic 2*Z*J*P*N*C*Q of the descriptors the calls carried.
        # An eager step is CPU-bound (3 400 launches x ~20 us of host work): a stream that drains faster than it is fed makes every
        # event pair also time the host gap between "record" and the launch behind it.  So the GPU is parked on a 30 ms spin
        # first (the host runs ~1 000 launches ahead and stays ahead), and the side streams are off so that kernels do not share
        # the SMs while they are being timed one by one.
        from easevoice_trainer_b200 import models as _models
        _ss, _models.SIDE_STREAMS = _models.SIDE_STREAMS, False
        try:
            torch.cuda._sleep(int(0.03 * 1.9e9))
            ops.profile_begin()
            st.step(batch, collectives=False)      # rank 0 alone: the profiled step must not enter the gradient all-reduces
            prof = ops.profile_end()
        finally:
            _models.SIDE_STREAMS = _ss
        tma_keys = [k for k in prof if "gemm_tma" in k or k.startswith("evk_gemm_tf32")]
        tma_ms = sum(prof[k]["ms"] for k in tma_keys)
        tma_fl = sum(prof[k]["flops"] for k in tma_keys)
        all_ms = sum(v["ms"] for v in prof.values())
        all_fl = sum(v["flops"] for v in prof.values())
        ach = tma_fl / (tma_ms * 1e-3) / 1e12
        table = kernel_table(ops, dev)
        top = sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[:14]
        extra["roofline"] = dict(bound="tensor", kernel="gemm_tma_kernel (TMA-fed persistent wgmma TF32 GEMM / implicit-GEMM conv: forward, data-gradient, "
                                                        "ConvTranspose-phase, strided-phase and weight-gradient launches)",
                                 achieved=ach, peak=tf_sus, unit="TFLOP/s", frac=ach / tf_sus,
                                 flops_per_step=tma_fl, ms_per_step=tma_ms, launches_per_step=sum(prof[k]["calls"] for k in tma_keys),
                                 share_of_step_time=tma_ms / all_ms, share_of_step_flops=tma_fl / all_fl,
                                 step_tflops=all_fl / (ms * 1e-3) / 1e12,
                                 peak_source=f"{src} bf16; the kernel computes in TF32 whose nominal peak is half of bf16",
                                 how="achieved = analytic flops of EVERY gemm_tma launch of one training step / the sum of their CUDA-event durations "
                                     "(events recorded on the launching stream around each call of an eager step run behind a 30 ms spin kernel so the host stays ahead, single stream, same process, after the timed region); "
                                     "share_of_step_time is against the event time of all library calls of that step (torch fill/add/copy kernels excluded)",
                                 by_call={k: dict(calls=v["calls"], ms=round(v["ms"], 3), tflops=(round(v["flops"] / (v["ms"] * 1e-3) / 1e12, 1) if v["flops"] else None))
                                          for k, v in top},
                                 layers=[{k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()} for r in table])
        # ---- fused mel kernel standalone: 16 x 10 s at the label rate, |X| + log-mel emitted
        Lw = batch["wav"].shape[1]
        nset, reps = 6, 3                                        # 6 x (wav 14 MB + |X| 23 MB + mel 3 MB) = 240 MB > L2
        wavs = [torch.rand(B_PER_GPU, Lw, device=dev) - 0.5 for _ in range(nset)]
        frames = B_PER_GPU * (Lw // HOP)
        def mel_burst():
            for _ in range(reps):
                for w in wavs:
                    ops.mel_frontend(w, st.bank, HOP, want_spec=True, want_mel=True)
        mel_burst()
        mel_ms = graph_time(mel_burst) / (nset * reps)
        alg_bytes = 4.0 * B_PER_GPU * Lw + frames * (1025 + 128) * 4.0     # SURVEY 8(d): 7172 B/frame with |X| emitted
        gbs = alg_bytes / (mel_ms * 1e-3) / 1e9
        # the same kernel on a dataset-preprocessing sized launch (256 x 10 s), where launch latency is amortised
        bigw = torch.rand(256, Lw, device=dev) - 0.5

        def mel_big():
            ops.mel_frontend(bigw, st.bank, HOP, want_spec=True, want_mel=True)
        mel_big()
        big_ms = graph_time(mel_big)
        big_frames = 256 * (Lw // HOP)
        big_gbs = (4.0 * bigw.numel() + big_frames * (1025 + 128) * 4.0) / (big_ms * 1e-3) / 1e9

        def mel_only():
            ops.mel_frontend(bigw, st.bank, HOP, want_spec=False, want_mel=True)
        mel_only()
        only_ms = graph_time(mel_only)
        only_gbs = (4.0 * bigw.numel() + big_frames * 128 * 4.0) / (only_ms * 1e-3) / 1e9
        del bigw
        extra["mel_roofline"] = dict(bound="hbm", kernel="mel_fwd_warp_kernel (|X| + log-mel emitted)", achieved=big_gbs, peak=hbm,
                                     unit="GB/s", frac=big_gbs / hbm, frames=big_frames, ms=big_ms, peak_source=src,
                                     how="one launch over 256 x 10 s (graph replay, 226 MB in + 408 MB out > L2)",
                                     batch16=dict(achieved=gbs, frac=gbs / hbm, frames=frames, ms=mel_ms,
                                                  how=f"{nset * reps} back-to-back launches of the training batch (16 x 10 s) over {nset} rotating buffer sets"),
                                     mel_only=dict(achieved=only_gbs, frac=only_gbs / hbm, ms=only_ms,
                                                   note="log-mel only (3 072 B/frame): FFT-arithmetic bound on the fp32 pipe"))
        line = dict(metric=METRIC, value=audio_s / (ms * 1e-3), unit=UNIT, n_gpus=world, steps=args.steps, warmup=args.warmup,
                    ms_per_step=ms, higher_is_better=True, scaling="weak", vs_baseline=None, dtype="tf32", data="synthetic",
                    config=workload_config(args.sr_label, world),
                    e2e=dict(value=audio_s / (ms_e2e * 1e-3), unit=UNIT, ms_per_step=ms_e2e, h2d_bytes_per_step=h2d,
                             d2h_bytes_per_step=8),
                    gpu_launches=launches, cuda_graph=not args.no_graph, clocks=clocks, losses=losses)
        line.update(extra)
    gpt = None
    if args.gpt and (world == 1 or args.gpt > 1):
        del st, net_g, net_d, batch
        torch.cuda.empty_cache()
        try:
            gpt = gpt_section(args, dev, rank, world)
        except Exception as e:                          # the headline line must survive a failure of the extra section
            import traceback
            traceback.print_exc()
            gpt = dict(error=repr(e)[:300])
    if rank == 0:
        line["gpt"] = gpt
        # The comparators below run LAST: the CPU arm leaves the host busy / memory-fragmented enough to slow the eager, event-timed
        # GPT profile above by 2x when it ran first (graph-replayed timings were never affected).
        extra = {}
        # ---- the same algorithm through stock PyTorch GPU kernels, whole optimisation step, same GPU: the ">= 10x the
        #      reference's 1-GPU PyTorch step" comparator of BASELINE.json, in the reference's as-shipped fp16-autocast regime
        #      and in fp32/TF32
        if not args.no_torch_port and world == 1:
            for key, amp in (("torch_gpu_port_fp16_autocast", True), ("torch_gpu_port", False)):
                try:
                    tms, tl = torch_gpu_port_step(dev, T, amp)
                    extra[key] = dict(ms_per_step=tms, value=B_PER_GPU * UTT_SECONDS / (tms * 1e-3), unit=UNIT, speedup_of_this_repo=tms / ms,
                                      loss_gen_all=tl,
                                      what="oracle port (the reference's algorithm) on stock PyTorch CUDA kernels, eager, B=16, forward + D backward + AdamW + "
                                           "G backward + AdamW, " + ("torch.autocast(float16) + GradScaler as the reference ships (fp16_run: true)" if amp
                                                                      else "fp32 storage with TF32 allowed (sovits.py:172-176)") + ", median of 5 steps")
                except Exception as e:                      # context only: never fail the benchmark because of it
                    extra[key] = dict(error=repr(e)[:300])
                torch.cuda.empty_cache()
        # ---- CPU baseline on the host's CPU cores: the full benchmark batch, whole optimisation step, bounded in time
        threads = cpu_threads()
        if not args.no_cpu_baseline and world == 1:                      # contract: rank 0 at N = 1 only
            Bc = args.cpu_batch if args.cpu_batch > 0 else B_PER_GPU
            sec, n_timed = cpu_reference_step(Bc, T, threads, 2, 0, budget_s=30.0)
            v = Bc * UTT_SECONDS / sec
            extra["cpu_baseline"] = dict(value=v, unit=UNIT, cores=threads, kind="port",
                                         sample=f"oracle port of sovits.py:459-525 (fwd, D bwd + AdamW, G bwd + AdamW; fp32), B={Bc} x 10 s, "
                                                f"T={T}, {n_timed} step(s), {sec:.1f} s/step")
        line.update(extra)
        emit(line)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def gpt_section(args, dev, rank, world):
    """BASELINE.json configs[1]: stage-1 AR-GPT (configs/gpt.yaml: 24 layers, d=512, 16 heads) training_step, batch 16 x
    (256 phonemes + 1024 semantic tokens) per GPU.  A step = one Lightning training_step (micro-batch fwd + bwd with
    dropout 0.1 as the reference hard-codes, gradient accumulation; ScaledAdam update on every 4th batch index)."""
    import torch
    import torch.distributed as dist
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    from easevoice_trainer_b200.train import gpt_step
    from easevoice_trainer_b200.configs import GPT_MODEL
    B, X, Y = 16, 256, 1024
    net = Text2SemanticDecoder({"model": GPT_MODEL}, seed=1234).to(dev).train()
    st = gpt_step.GptStep(net, world_size=world)
    host = gpt_step.synthetic_batch(B, X, Y, seed=4321 + rank, device="cpu")
    h2d = sum(v.numel() * v.element_size() for v in host.values())
    batch = {k: v.to(dev) for k, v in host.items()}
    batch["bert_feature"] = ops.to_channels_last(batch["bert_feature"]); batch["bert_channels_last"] = True
    l0 = ops.launches()
    st.batch_idx = 4                                  # an eager step that includes the optimizer update
    st.step(batch)
    launches = ops.launches() - l0
    torch.cuda.synchronize()
    peak_gb = torch.cuda.max_memory_allocated(dev) / 2**30
    run = st.step if args.no_graph else st.graph_step
    last = {}

    def resident():
        last["out"] = run(batch)

    def e2e():
        b = {k: v.to(dev, non_blocking=True) for k, v in host.items()}
        b["bert_feature"] = ops.to_channels_last(b["bert_feature"]); b["bert_channels_last"] = True
        out = run(b)
        last["host"] = torch.stack([out[0].reshape(()), out[1].reshape(())]).cpu()

    def timed(fn, steps):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms) / steps
    for _ in range(max(args.warmup, 3)):
        resident()
    st.batch_idx = 1
    steps = args.steps                                 # micro-batches; every 4th runs the optimizer update (accumulate 4)
    ms = timed(resident, steps)
    st.batch_idx = 1
    for _ in range(2):
        e2e()
    st.batch_idx = 1
    ms_e2e = timed(e2e, steps)
    # optimizer update alone
    st.batch_idx = 4
    def opt_only():
        st._ograph.replay() if not args.no_graph else st.opt.step()
    ms_opt = timed(opt_only, 4)
    # dominant kernels of this step from one profiled eager micro-batch (same accounting as the stage-2 roofline)
    roof = cpu = None
    if rank == 0:
        hbm, tf_burst, tf_sus, src = peaks()
        st.batch_idx = 1
        ops.profile_begin()
        st.step(batch)
        prof = ops.profile_end()
        keys = [k for k in prof if "gemm_tma" in k or k.startswith("evk_gemm_tf32")]
        g_ms, g_fl = sum(prof[k]["ms"] for k in keys), sum(prof[k]["flops"] for k in keys)
        all_ms = sum(v["ms"] for v in prof.values())
        attn = {k: round(v["ms"], 3) for k, v in prof.items() if "flash" in k}
        roof = dict(bound="tensor", kernel="gemm_tma_kernel (six Linear layers per block: forward, data gradient, weight gradient)", achieved=g_fl / (g_ms * 1e-3) / 1e12,
                    peak=tf_sus, unit="TFLOP/s", frac=g_fl / (g_ms * 1e-3) / 1e12 / tf_sus,
                    share_of_step_time=g_ms / all_ms, attention_ms=attn, attention_share_of_step_time=sum(attn.values()) / all_ms,
                    peak_source=f"{src} bf16 (TF32 nominal = half)",
                    how="analytic flops of every gemm_tma launch of one micro-batch / the sum of their CUDA-event durations (eager step, events around each library call)")
        if not args.no_cpu_baseline and world == 1:
            cpu = gpt_cpu_baseline(B, X, Y)
    tok = world * B * Y
    flops = 6.0 * (B * (X + Y)) * (24 * (4 * 512 * 512 + 2 * 512 * 2048)) + 6.0 * B * Y * 512 * 1025 + 6.0 * B * X * 1024 * 512 \
        + 24 * 3.5 * 4.0 * B * 16 * (X + Y) ** 2 * 32 * 0.62     # attention: fwd + 2.5x bwd (S recomputed twice), ~62% of L^2 visible
    return dict(metric="stage-1 AR-GPT training_step semantic-tokens/sec", value=tok / (ms * 1e-3), unit="semantic-tokens/s",
                ms_per_step=ms, steps=steps, config=dict(workload=f"gpt_step_B{B}_X{X}_Y{Y}_L24_d512_h16", dropout=0.1, accumulate=4,
                                                         optimizer="ScaledAdam (flat, 3 launches)", parallelism=f"dp{world}"),
                e2e=dict(value=tok / (ms_e2e * 1e-3), unit="semantic-tokens/s", ms_per_step=ms_e2e, h2d_bytes_per_step=h2d, d2h_bytes_per_step=8),
                optimizer_ms=ms_opt, gpu_launches_per_step_with_update=launches, peak_mem_gb=peak_gb,
                model_tflops=flops * world / (ms * 1e-3) / 1e12, cuda_graph=not args.no_graph, roofline=roof, cpu_baseline=cpu,
                loss=float(last["out"][0]), acc=float(last["out"][1]))


def gpt_cpu_baseline(B, X, Y, Bc=2):
    """the reference's algorithm (oracle port of t2s_model.py:431-490 forward_old + backward, fp32) on the host cores:
    bounded sample of Bc sequences of the same X / Y / depth."""
    import torch
    from oracle import gpt_oracle
    threads = cpu_threads()
    torch.set_num_threads(threads)
    m = dict(gpt_oracle.GPT_MODEL)
    P = {k: v.clone().requires_grad_(True) for k, v in gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), 1234).items()}
    x, xl, y, yl, bert = gpt_oracle.synthetic_gpt_batch(Bc, X, Y, 5, False)
    t0 = time.perf_counter()
    loss = gpt_oracle.forward_old(P, x, xl, y, yl, bert, m)[0]
    loss.backward()
    sec = time.perf_counter() - t0
    return dict(value=Bc * Y / sec, unit="semantic-tokens/s", cores=threads, kind="port",
                sample=f"oracle port of forward_old + backward (24 layers, fp32, dropout off), B={Bc}, X={X}, Y={Y}, 1 cold micro-batch, {sec:.1f} s")


def config5_section(args, dev):
    """BASELINE.json configs[4]: HiFi-GAN generator + MPD/MSD + losses only, batch 32 x 1 s at the 48 kHz label (z [32,192,75] ->
    y_hat [32,1,48000]), with the multi-resolution STFT loss as the opt-in extension (bs_roformer.py:565-581).  One "step" =
    generator forward, discriminators on (y, y_hat), GAN + feature-matching + MR-STFT losses, backward through everything
    (weight gradients of G and D, d z).  Reports the step time and the per-layer sweep of SURVEY 8(d): every contraction
    launch of the step with its shape, device time, achieved TFLOP/s and algorithmic GB/s."""
    import torch
    from easevoice_trainer_b200 import ops, models, configs
    hps = configs.load_s2_config()
    torch.manual_seed(1234)
    net_g = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                                  n_speakers=hps["data"]["n_speakers"], **hps["model"]).to(dev).train()
    net_d = models.MultiPeriodDiscriminator(False).to(dev).train()
    B, T = 32, 75
    g = torch.Generator().manual_seed(5)
    z = (torch.randn(B, T, 192, generator=g)).to(dev).requires_grad_(True)
    ge = (torch.randn(B, 1, 512, generator=g) * 0.5).to(dev)
    y = (torch.rand(B, T * 640, 1, generator=g) - 0.5).to(dev)
    gp = [p_ for n, p_ in net_g.named_parameters() if n.startswith("dec.")]
    dp = list(net_d.parameters())

    def step(mr=True):
        net_g.begin_pack()
        try:
            yh = net_g._generator(z, ge)
        finally:
            net_g.end_pack()
        outs = net_d.forward_cl(y, yh)
        lg = lf = ld = 0.0
        for logit, fmap in outs:
            lg = lg + ops.mean_sq_one_minus(logit[B:])
            ld = ld + ops.mean_sq_one_minus(logit[:B]) + ops.mean_sq(logit[B:])
            for f in fmap:
                lf = lf + ops.mean_abs_diff(f[B:], f[:B])
        loss = lg + 2.0 * lf + ld
        if mr:
            loss = loss + ops.mrstft_loss(yh.reshape(B, -1), y.reshape(B, -1))
        torch.autograd.grad(loss, [z] + gp + dp)
        return loss.detach()
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    out = {}
    for key, mr in (("with_mrstft", True), ("without_mrstft", False)):
        st_ = lambda: step(mr)
        st_()
        ms = graph_time(st_)
        out[key] = dict(ms_per_step=ms, audio_s_per_s=B * 1.0 / (ms * 1e-3))
    # per-launch sweep from one profiled eager step
    rows = []
    orig = ops._run_desc

    def rec_desc(fn, d):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        orig(fn, d)
        e1.record()
        rows.append((fn, dict(Z=d.Z, C=d.C, N=d.N, Q=d.Q, J=d.J, P=d.P, stride=d.is_, os=d.os_, H=d.H), e0, e1,
                     2.0 * d.Z * d.J * d.P * d.N * d.C * d.Q, 4.0 * d.Z * (d.J * d.P * d.N + d.Tin * d.P * d.C) + 4.0 * d.Q * d.N * d.C))
    ops._run_desc = rec_desc
    try:
        step(True)
    finally:
        ops._run_desc = orig
    torch.cuda.synchronize()
    agg = {}
    for fn, shp, e0, e1, fl, by in rows:
        k = (fn,) + tuple(shp.items())
        a = agg.setdefault(k, dict(call=fn, **shp, launches=0, ms=0.0, flops=0.0, bytes=0.0))
        a["launches"] += 1; a["ms"] += e0.elapsed_time(e1); a["flops"] += fl; a["bytes"] += by
    table = sorted(agg.values(), key=lambda a: -a["ms"])
    for a in table:
        a["tflops"] = round(a["flops"] / (a["ms"] * 1e-3) / 1e12, 1)
        a["gbs"] = round(a["bytes"] / (a["ms"] * 1e-3) / 1e9, 0)
        a["ms"] = round(a["ms"], 4)
        del a["flops"], a["bytes"]
    out["layers"] = table[:60]
    out["config"] = dict(workload="vocoder_only_B32x1s_sr48000 (z [32,192,75] -> y_hat [32,1,48000])", mrstft_windows=[4096, 2048, 1024, 512, 256], mrstft_hop=147)
    out["how"] = ("step: CUDA-graph replay between CUDA events; layers: conv-family launches of one eager step (forward, data-gradient phases; weight gradients "
                  "of the TMA path are listed by the bench roofline instead), grouped by shape, device time from events around each launch; GB/s = (input + output "
                  "+ weight bytes, once) / time")
    return out


def emit(line):
    """write the one JSON line to the REAL stdout (fd 1 is pointed at stderr while the benchmark runs so that library
    banners -- e.g. NCCL's version line -- cannot pollute the result stream)."""
    os.write(_REAL_STDOUT, (json.dumps(line) + "\n").encode())


_REAL_STDOUT = 1


def main():
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--sr-label", type=int, default=22050, help="BASELINE.json quotes 10 s @ 22.05 kHz; 32000 = native s2.json rate")
    ap.add_argument("--cpu-batch", type=int, default=0, help="utterances per step of the CPU arm (0 = the benchmark batch, 16)")
    ap.add_argument("--cpu-budget", type=float, default=200.0, help="--impl reference: wall-time bound (s) of its timed region")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-torch-port", action="store_true")
    ap.add_argument("--only-gpt", action="store_true", help="profiling aid: run just the stage-1 AR-GPT section and print its object")
    ap.add_argument("--gpt", type=int, default=2, help="2 (default): also time the stage-1 AR-GPT step at every N; 1: at N=1 only; 0: skip")
    ap.add_argument("--config", type=int, default=3, help="3 (default): the stage-2 step (BASELINE configs 3/4); 5: vocoder-only per-layer sweep with the MR-STFT loss")
    ap.add_argument("--no-graph", action="store_true", help="launch every kernel from Python instead of replaying the captured CUDA graph")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's losses and a seeded sample of the updated parameters as DIR/<name>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)
    args.warmup = max(args.warmup, 3)
    return run_ours(args)


if __name__ == "__main__":
    sys.exit(main())
