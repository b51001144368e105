"""Stage-1 training throughput of the GPTTrain loop on a seeded synthetic project: the eager step at the collate's shapes
against GptStep.train_step (padded to the 32-token grid, one CUDA graph per shape), alternated epoch by epoch in one
process, with the default model (24 layers) and batch size (12).  A third arm runs train_step with the DataLoader in two
worker processes, to show whether the in-process loader stalls the replayed step.

The project has --items utterances of 2-12 s (50-300 semantic tokens, 8-16 phonemes per second of audio) with BERT features,
so the duration-bucketed sampler yields ragged batches of many shapes.  Per arm and epoch it reports semantic tokens/s (real
tokens, not padding; wall clock over the epoch, every step ends in the trainer's host read of loss and accuracy), the mean
time per step spent waiting for the loader, and the graph captures, replays and eager fallbacks.  The first epoch of every
arm is warm-up and is not counted.  Prints one JSON line with the card's name and power limit.

    python tools/bench_gpt_train.py [--items 480] [--rounds 3] [--dpo]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from easevoice_trainer_b200 import lib, ops  # noqa: E402
from easevoice_trainer_b200.train import data_gpt, gpt_step  # noqa: E402
from easevoice_trainer_b200.train.gpt import GPTTrain, GPTTrainParams  # noqa: E402


def write_project(root, items, seed):
    inp = os.path.join(root, "in")
    os.makedirs(os.path.join(inp, "3-bert"))
    g = torch.Generator().manual_seed(seed)
    with open(os.path.join(inp, "2-name2text.txt"), "w") as f2, open(os.path.join(inp, "6-name2semantic.tsv"), "w") as f6:
        f6.write("item_name\tsemantic_audio\n")
        for i in range(items):
            nsem = int(torch.randint(50, 301, (1,), generator=g))
            nph = max(int(nsem / 25 * float(torch.empty(1).uniform_(8, 16, generator=g))), 4)
            f2.write(f"utt{i}\t" + " ".join(f"p{int(v)}" for v in torch.randint(0, 732, (nph,), generator=g)) + "\tw2p\ttext\n")
            f6.write(f"utt{i}\t" + " ".join(str(int(v)) for v in torch.randint(0, 1024, (nsem,), generator=g)) + "\n")
            torch.save(torch.randn(1024, nph, generator=g), os.path.join(inp, "3-bert", f"utt{i}.pt"))
    return inp


class Arm:
    def __init__(self, name, trainer, ds, dev, graphs, workers, dpo):
        t = trainer.config["train"]
        self.name, self.dev, self.graphs = name, dev, graphs
        self.step = gpt_step.GptStep(trainer._build(dev), dpo=dpo)
        bs = t["batch_size"] // 2 if dpo else t["batch_size"]
        self.sampler = data_gpt.DistributedBucketSampler(ds, 1, 0, batch_size=bs)
        self.loader = torch.utils.data.DataLoader(ds, batch_size=bs, sampler=self.sampler, collate_fn=ds.collate, num_workers=workers,
                                                  pin_memory=True, persistent_workers=workers > 0)
        self.epochs = []

    def epoch(self, e):
        self.sampler.set_epoch(e)
        self.step.batch_idx = 0
        before = dict(self.step.stats)
        tokens, wait, steps = 0, 0.0, 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        it = iter(self.loader)
        while True:
            w0 = time.perf_counter()
            host = next(it, None)
            wait += time.perf_counter() - w0
            if host is None:
                break
            if self.graphs:
                loss, acc = self.step.train_step(self.step.prepare(host, self.dev))
            else:
                batch = {k: v.to(self.dev, non_blocking=True) for k, v in host.items() if k != "ids"}
                loss, acc = self.step.step(batch)
            float(loss), float(acc)                      # GPTTrain writes both to stdout after every step
            tokens += int(host["semantic_ids_len"].sum())
            steps += 1
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        st = {k: self.step.stats[k] - before[k] for k in before} if self.graphs else dict(captures=0, replays=0, eager=steps)
        self.epochs.append(dict(tokens_per_s=tokens / dt, ms_per_step=1e3 * dt / steps, loader_wait_ms_per_step=1e3 * wait / steps,
                                steps=steps, **st))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=480)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dpo", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    lib.init()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    with tempfile.TemporaryDirectory() as td:
        inp = write_project(td, args.items, 1234)
        params = GPTTrainParams(if_dpo=args.dpo, gpu_ids="0", model_path="", train_input_dir=inp, output_model_name="bench",
                                project_dir=td)
        trainer = GPTTrain(params)
        ds = data_gpt.Text2SemanticDataset(trainer.config["train_phoneme_path"], trainer.config["train_semantic_path"],
                                           max_sec=trainer.config["data"]["max_sec"], phoneme_table={f"p{i}": i for i in range(732)})
        ops.manual_seed(trainer.config["train"]["seed"])
        arms = [Arm("eager step", trainer, ds, dev, False, 0, args.dpo), Arm("train_step", trainer, ds, dev, True, 0, args.dpo),
                Arm("train_step, 2 loader workers", trainer, ds, dev, True, 2, args.dpo)]
        for r in range(args.rounds + 1):
            for a in arms:
                a.epoch(r)
                print(a.name, r, json.dumps(a.epochs[-1]), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip(), batch_size=trainer.config["train"]["batch_size"], dpo=args.dpo, items=len(ds), rounds=args.rounds,
               arms={a.name: dict(warm=a.epochs[1:], warmup=a.epochs[0],
                                  tokens_per_s=[round(e["tokens_per_s"]) for e in a.epochs[1:]]) for a in arms})
    base = sum(e["tokens_per_s"] for e in arms[0].epochs[1:])
    res["speedup_train_step"] = sum(e["tokens_per_s"] for e in arms[1].epochs[1:]) / base
    res["speedup_train_step_workers"] = sum(e["tokens_per_s"] for e in arms[2].epochs[1:]) / base
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
