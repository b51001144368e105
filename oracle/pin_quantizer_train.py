"""Pin the trainable semantic quantizer (freeze_quantizer: false) against the UNMODIFIED reference and write
tests/golden/s2_quantizer_train.pt.  Needs EVK_REFERENCE (a checkout of the reference); no test imports this module.

    EVK_REFERENCE=/path/to/easevoice-trainer python -m oracle.pin_quantizer_train

Small config (D = 64 channels, K = 128 codes, B = 3, T = 400 frames, so 600 rows: more than the 500 k-means samples):
ssl_proj (Conv1d(D, D, 2, stride 2)) -> core_vq.VectorQuantization in training mode -> nearest x2 upsample, and the loss
sum(G * quantized) + kl_ssl, for three forwards from a zero codebook with inited = 0.  core_vq.sample_vectors is wrapped to
record the k-means sample indices; the inputs come from `vq_train_oracle.pin_inputs` (seeded).  Also pinned: k-means on small-integer samples (every distance and mean exact, many
duplicate means, so the tie rule decides), and that dead-code expiry leaves no trace (threshold_ema_dead_code 0 vs 2).
"""
import os
import sys

import torch
import torch.nn.functional as F

from oracle import vq_train_oracle as O

REF = os.environ.get("EVK_REFERENCE", "")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "s2_quantizer_train.pt")
CFG = dict(B=3, D=64, K=128, T=400, steps=3, seed=20261016)


def import_core_vq():
    sys.path.insert(0, REF)
    from src.easevoice.module import core_vq
    recorded = []

    def sample_vectors(samples, num):            # core_vq.py:60-68, recording the indices
        n = samples.shape[0]
        idx = torch.randperm(n)[:num] if n >= num else torch.randint(0, n, (num,))
        recorded.append(idx.clone())
        return samples[idx]
    core_vq.sample_vectors = sample_vectors
    return core_vq, recorded


def run_reference(core_vq, recorded, threshold):
    c = CFG
    w0, b0, ssls, ups = O.pin_inputs(c)
    ssl_proj = torch.nn.Conv1d(c["D"], c["D"], 2, stride=2)
    with torch.no_grad():
        ssl_proj.weight.copy_(w0)
        ssl_proj.bias.copy_(b0)
    vq = core_vq.VectorQuantization(dim=c["D"], codebook_size=c["K"], kmeans_iters=50, threshold_ema_dead_code=threshold)
    vq.train()
    torch.manual_seed(c["seed"])
    del recorded[:]
    steps = []
    for ssl, up in zip(ssls, ups):
        ssl_proj.zero_grad()
        x = ssl_proj(ssl)
        q, codes, loss = vq(x)
        qu = F.interpolate(q, size=int(q.shape[-1] * 2), mode="nearest")
        ((qu * up).sum() + loss.mean()).backward()
        cb = vq._codebook
        steps.append(dict(codes=codes.detach().clone(), kl_ssl=loss.detach().reshape(()).clone(),
                          buffers={k: getattr(cb, k).detach().clone() for k in ("embed", "embed_avg", "cluster_size", "inited")},
                          dweight=ssl_proj.weight.grad.clone(), dbias=ssl_proj.bias.grad.clone()))
    return dict(kmeans_idx=recorded[0].clone(), steps=steps)


def integer_kmeans(core_vq, recorded):
    g = torch.Generator().manual_seed(7)
    points = torch.randint(-3, 4, (8, 16), generator=g).float()
    samples = points[torch.randint(0, 8, (40,), generator=g)]
    torch.manual_seed(11)
    del recorded[:]
    means, bins = core_vq.kmeans(samples, 64, 50)
    return dict(samples=samples, idx=recorded[0].clone(), means=means, bins=bins)


def main():
    assert os.path.isdir(os.path.join(REF, "src")), "set EVK_REFERENCE to a checkout of the reference"
    core_vq, recorded = import_core_vq()
    run = run_reference(core_vq, recorded, threshold=2)
    run0 = run_reference(core_vq, recorded, threshold=0)
    for a, b in zip(run["steps"], run0["steps"]):              # expire_codes_ is overwritten by embed_normalized
        for k in a["buffers"]:
            assert torch.equal(a["buffers"][k], b["buffers"][k]), k
        assert torch.equal(a["codes"], b["codes"])
    ik = integer_kmeans(core_vq, recorded)
    m, bins, _ = O.kmeans(ik["samples"], 64, 50, ik["idx"])
    assert torch.equal(m, ik["means"]) and torch.equal(bins, ik["bins"]), "oracle k-means != reference k-means"
    gold = dict(cfg=CFG, run=run, kmeans_int=ik, expiry_inert=True)
    torch.save(gold, OUT)
    print("wrote", os.path.normpath(OUT), "kl_ssl", [float(s["kl_ssl"]) for s in run["steps"]])


if __name__ == "__main__":
    main()
