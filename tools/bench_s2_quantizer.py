"""Stage-2 graph step time with the frozen and with the trainable semantic quantizer (freeze_quantizer true / false), at the
benchmark's shape (B = 16 utterances of 10 s), alternated in one process.  Prints one JSON line with the card's name and
power limit.

    python tools/bench_s2_quantizer.py [--steps 20] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from easevoice_trainer_b200 import configs, lib, models, ops  # noqa: E402
from easevoice_trainer_b200.train import s2_step  # noqa: E402


def make(freeze, dev, host):
    hps = configs.load_s2_config()
    hps["model"]["freeze_quantizer"] = freeze
    torch.manual_seed(hps["train"]["seed"])
    net_g = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                                  n_speakers=hps["data"]["n_speakers"], **hps["model"]).to(dev).train()
    net_d = models.MultiPeriodDiscriminator(hps["model"]["use_spectral_norm"]).to(dev).train()
    st = s2_step.S2Step(net_g, net_d, hps["train"], hps["data"])
    batch = s2_step.to_device_batch(host, dev, st.bank, vq_frames=host["ssl"].shape[2] if not freeze else None)
    st.step(batch)                       # eager (the unfrozen one k-means-initialises its codebook here)
    st.graph_step(batch)                 # capture
    return st, batch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib.init()
    dev = torch.device("cuda", 0)
    ops.manual_seed(1234)
    host = s2_step.synthetic_batch(bench.B_PER_GPU, bench.frames_for(22050), bench.TEXT_LEN, dev, seed=1234)
    arms = {"frozen": make(True, dev, host), "unfrozen": make(False, dev, host)}
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, (st, batch) in arms.items():
            for _ in range(3):
                st.graph_step(batch)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                st.graph_step(batch)
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / args.steps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    fz, uf = min(ms["frozen"]), min(ms["unfrozen"])
    print(json.dumps(dict(metric="s2_step_ms_quantizer", B=bench.B_PER_GPU, frames=int(host["ssl"].shape[2]), frozen_ms=round(fz, 3),
                          unfrozen_ms=round(uf, 3), overhead_pct=round(100.0 * (uf - fz) / fz, 2),
                          rounds={k: [round(v, 3) for v in vs] for k, vs in ms.items()}, card=card)))


if __name__ == "__main__":
    main()
