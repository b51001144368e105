"""CPU restatement of the trainable semantic quantizer (freeze_quantizer: false): ssl_proj, k-means initialisation, EMA
codebook update, straight-through value with the nearest x2 upsample and the commitment loss (the reference's core_vq.py:71-93,
141-149, 203-228, 301-318 and models.py:917-927).  fp32 torch on the CPU; rows are in the reference collate's (batch, frame)
order, and only the first `rows_ref` frames of every batch row take part.
"""
import torch
import torch.nn.functional as F

DECAY, EPS, MAX_KMEANS_SAMPLES = 0.99, 1e-5, 500


def pin_inputs(cfg):
    """the pinned run's inputs, generated from its seed: ssl_proj weight / bias, and per forward ssl [B, D, T] and the
    upstream gradient G [B, D, T] of the loss sum(G * quantized_up) + kl_ssl"""
    g = torch.Generator().manual_seed(cfg["seed"])
    w = torch.randn(cfg["D"], cfg["D"], 2, generator=g) * 0.1
    b = torch.randn(cfg["D"], generator=g) * 0.1
    ssls = [torch.randn(cfg["B"], cfg["D"], cfg["T"], generator=g) for _ in range(cfg["steps"])]
    ups = [torch.randn(cfg["B"], cfg["D"], cfg["T"], generator=g) for _ in range(cfg["steps"])]
    return w, b, ssls, ups


def kmeans(samples, K, iters, idx):
    """core_vq.kmeans with the initial means samples[idx] -> (means [K, D], bins int64 [K], buckets of the last iteration).
    Assignment: argmax of -sum (s - m)^2 in direct-difference form, lowest index on ties."""
    samples = samples[:MAX_KMEANS_SAMPLES]
    means = samples[idx].clone()
    K = means.shape[0]
    for _ in range(iters):
        dists = -((samples[:, None, :] - means[None, :, :]) ** 2).sum(-1)
        buckets = dists.max(dim=-1).indices
        bins = torch.bincount(buckets, minlength=K)
        new = torch.zeros_like(means).index_add_(0, buckets, samples)
        new = new / bins.clamp(min=1)[:, None]
        means = torch.where((bins == 0)[:, None], means, new)
    return means, bins, buckets


def nearest(x, embed):
    """EuclideanCodebook.quantize (expanded form)."""
    dist = -(x.pow(2).sum(1, keepdim=True) - 2 * x @ embed.t() + embed.pow(2).sum(1)[None, :])
    return dist.max(dim=-1).indices


def ema(buffers, x, codes):
    """training-mode EMA of cluster_size / embed_avg and the normalised embed (core_vq.py:218-226) -> new buffers."""
    K = buffers["embed"].shape[0]
    onehot = F.one_hot(codes, K).float()
    cs = buffers["cluster_size"] * DECAY + onehot.sum(0) * (1 - DECAY)
    ea = buffers["embed_avg"] * DECAY + (x.t() @ onehot).t() * (1 - DECAY)
    n = cs.sum()
    norm = (cs + EPS) / (n + K * EPS) * n
    return dict(embed=ea / norm[:, None], embed_avg=ea, cluster_size=cs, inited=buffers["inited"].clone())


def step(ssl, weight, bias, buffers, upstream, kmeans_idx=None, rows_ref=None, kmeans_iters=50):
    """One training-mode forward + backward of ssl_proj -> quantizer -> nearest x2, with loss
    sum(upstream * quantized_up) + kl_ssl.  ssl [B, D, T] (T even), upstream [B, D, T].
    -> dict(codes [B, rows_ref], kl_ssl, buffers (after the EMA), dweight, dbias, kmeans_idx)."""
    B, D, T = ssl.shape
    T2 = T // 2
    rows_ref = T2 if rows_ref is None else rows_ref
    w = weight.clone().requires_grad_(True)
    b = bias.clone().requires_grad_(True)
    xc = F.conv1d(ssl[:, :, :2 * rows_ref], w, b, stride=2)                 # [B, D, rows_ref]
    x = xc.transpose(1, 2).reshape(-1, D)
    buf = {k: v.clone() for k, v in buffers.items()}
    if float(buf["inited"]) == 0:
        xs = x.detach()[:MAX_KMEANS_SAMPLES]
        means, bins, _ = kmeans(xs, buf["embed"].shape[0], kmeans_iters, kmeans_idx)
        buf.update(embed=means.clone(), embed_avg=means.clone(), cluster_size=bins.float(), inited=torch.ones(1))
    codes = nearest(x.detach(), buf["embed"])
    q = buf["embed"][codes]
    buf = ema(buf, x.detach(), codes)
    qst = x + (q - x).detach()
    kl = F.mse_loss(qst.detach(), x)
    up = qst.reshape(B, rows_ref, D).repeat_interleave(2, dim=1).transpose(1, 2)      # nearest x2: [B, D, 2 rows_ref]
    loss = (up * upstream[:, :, :2 * rows_ref]).sum() + kl
    loss.backward()
    return dict(codes=codes.reshape(B, rows_ref), kl_ssl=kl.detach(), buffers=buf, dweight=w.grad, dbias=b.grad,
                kmeans_idx=kmeans_idx)
