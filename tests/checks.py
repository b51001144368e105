"""GPU parity checks: every libevk kernel family and the assembled stage-2 step against the CPU oracle
(oracle/ = torch-fp32 restatement of the reference, pinned by oracle/pin_against_reference.py).

Each check returns a list of (name, error, tolerance) triples; tests/test_gpu_parity.py asserts them,
tests/run_gpu_checks.py prints all of them without stopping.

Tolerance table (stated once, used everywhere; relative L2 unless noted):
  TOL_F32   = 2e-5   pure fp32 CUDA-core kernels
  TOL_TC    = 1e-3   "TF32-class" gate of BASELINE.md: the result of ONE tensor-core contraction on a linear path
                     (y, dx, dW, dbias of a conv / linear / attention forward; 10-bit operand mantissa, fp32 accumulate)
  TOL_TC2   = 2e-3   the result of TWO chained contractions inside one op (attention dq/dk/dv: S is recomputed, then
                     dS.K; weight-norm dv/dg: dW then the norm projection)
  TOL_NET   = 3e-3   activations / losses at the END of an assembled network (10-100 tensor-core launches deep)
  KINK_TOL  = 2.5e-2 any gradient that crossed a (leaky-)ReLU: compared across two forward roundings, pre-activations
                     within rounding distance of 0 flip their derivative (slope 0.1 <-> 1); 3xTF32 mode collapses it
                     (test_precise_mode_tightens_*), i.e. it is rounding, not indexing
  NET_GRAD  = 1e-2 global / 5e-2 worst single tensor: parameter gradients of the assembled stage-2 networks
                     ("BF16-class" gate of BASELINE.md for the global number); the GPT uses KINK_TOL global
  integer results (VQ codes, slice ids, masks, targets) must be bit-exact.
"""
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import mel_oracle, s2_oracle, gpt_oracle  # noqa: E402  (checker only)

TOL_TC = 1e-3
TOL_TC2 = 2e-3
TOL_NET = 3e-3
TOL_F32 = 2e-5
KINK_TOL = 2.5e-2          # gradients through ReLU-type kinks under TF32 forward rounding (see check_conv)
NET_GRAD_GLOBAL, NET_GRAD_TENSOR = 1e-2, 5e-2
PRECISE_MODE = [False]     # set by the caller when the library runs in 3xTF32 mode
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


def cl(x):      # [B,C,T] cpu -> [B,T,C] cuda
    return x.transpose(1, 2).contiguous().to(DEV)


def cf(x):      # [B,T,C] cuda -> [B,C,T] cpu
    return x.detach().transpose(1, 2).contiguous().cpu()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------
def check_conv():
    from easevoice_trainer_b200 import ops
    out = []
    cfgs = [
        # name, B, Tin, C, N, Q, stride, pad, dil, P, G, act, res, masks
        ("resblock k3 d1", 2, 97, 32, 32, 3, 1, 1, 1, 1, 1, 1, True, False),
        ("resblock k11 d5", 2, 300, 64, 64, 11, 1, 25, 5, 1, 1, 1, False, False),
        ("resblock k7 d3 c16", 2, 515, 16, 16, 7, 1, 9, 3, 1, 1, 0, True, False),
        ("conv_pre k7 192->512", 3, 32, 192, 512, 7, 1, 3, 1, 1, 1, 0, False, False),
        ("wn in_layer k5 +mask", 3, 70, 192, 384, 5, 1, 2, 1, 1, 1, 0, False, True),
        ("ffn k3 192->768 relu", 2, 61, 192, 768, 3, 1, 1, 1, 1, 1, 2, False, True),
        ("linear 1025->192", 2, 50, 1025, 192, 1, 1, 0, 1, 1, 1, 0, False, True),
        ("linear 96->192", 2, 50, 96, 192, 1, 1, 0, 1, 1, 1, 0, False, False),
        ("ssl_proj k2 s2", 2, 50, 768, 768, 2, 2, 0, 1, 1, 1, 0, False, False),
        ("discP 32->128 s3 p=2", 2, 119, 32, 128, 5, 3, 2, 1, 2, 1, 1, False, False),
        ("discP 128->512 s3 p=11", 2, 40, 128, 512, 5, 3, 2, 1, 11, 1, 1, False, False),
        ("discP 1024->1024 s1 p=3", 2, 23, 1024, 1024, 5, 1, 2, 1, 3, 1, 1, False, False),
        ("discP 1->32 s3 p=5 (direct)", 2, 200, 1, 32, 5, 3, 2, 1, 5, 1, 1, False, False),
        ("discP post 1024->1 p=7", 2, 23, 1024, 1, 3, 1, 1, 1, 7, 1, 0, False, False),
        ("discS 1->16 k15 (direct)", 2, 1000, 1, 16, 15, 1, 7, 1, 1, 1, 1, False, False),
        ("discS 16->64 k41 s4 g4 (direct)", 2, 1000, 16, 64, 41, 4, 20, 1, 1, 4, 1, False, False),
        ("discS 256->1024 k41 s4 g64 (direct)", 2, 130, 256, 1024, 41, 4, 20, 1, 1, 64, 1, False, False),
        ("conv_post 16->1 k7 tanh", 2, 700, 16, 1, 7, 1, 3, 1, 1, 1, 3, False, False),
        # large enough for the TMA implicit-GEMM path (csrc/gemm_tma.cu conv mode): taps via box coordinates, OOB = padding
        ("TMA resblock k11 d1 128ch +res", 3, 1500, 128, 128, 11, 1, 5, 1, 1, 1, 1, True, False),
        ("TMA resblock k7 d5 64ch", 2, 2100, 64, 64, 7, 1, 15, 5, 1, 1, 1, False, False),
        ("TMA conv_pre k7 192->512", 5, 500, 192, 512, 7, 1, 3, 1, 1, 1, 0, False, False),
        ("TMA discP 512->1024 k5 s1 p=3", 3, 310, 512, 1024, 5, 1, 2, 1, 3, 1, 1, False, False),
        ("TMA k3 32->96 (C tail zero-fill)", 2, 1100, 36, 96, 3, 1, 1, 1, 1, 1, 0, False, False),
        # strided forwards through the phase split + the multi-source tap sum; dgrad phases use the os/o0 output mapping
        ("TMA discP 128->512 k5 s3 p=2 (phased)", 4, 1000, 128, 512, 5, 3, 2, 1, 2, 1, 1, False, False),
        ("TMA discP 32->128 k5 s3 p=5 (phased)", 3, 410, 32, 128, 5, 3, 2, 1, 5, 1, 0, False, False),
        ("TMA ssl_proj k2 s2 768->768 (phased)", 6, 700, 768, 768, 2, 2, 0, 1, 1, 1, 0, False, False),
        ("TMA k41 s4 64->64 (phased)", 3, 3000, 64, 64, 41, 4, 20, 1, 1, 1, 1, False, False),
    ]
    for i, (name, B, Tin, C, N, Q, stride, pad, dil, P, G, act, use_res, masks) in enumerate(cfgs):
        g = _gen(100 + i)
        x = torch.randn(B, C, Tin * P if P == 1 else Tin, P, generator=g) if P > 1 else torch.randn(B, C, Tin, generator=g)
        v = torch.randn(N, C // G, Q, generator=g) / math.sqrt(C // G * Q)
        gg = 0.5 + torch.rand(N, 1, 1, generator=g)
        bias = torch.randn(N, generator=g) * 0.1
        lens = torch.tensor([Tin] + [max(Tin - 7 * (b + 1), 3) for b in range(B - 1)])
        xr = x.clone().requires_grad_(True)
        vr, gr, br = v.clone().requires_grad_(True), gg.clone().requires_grad_(True), bias.clone().requires_grad_(True)
        w = vr * (gr / vr.flatten(1).norm(dim=1).view(-1, 1, 1))
        xin = xr
        if masks:
            m = (torch.arange(Tin)[None, :] < lens[:, None]).float().unsqueeze(1)
            xin = xr * m
        if P == 1:
            y = F.conv1d(xin, w, br, stride, pad, dil, G)
        else:
            y = F.conv2d(xin, w.unsqueeze(-1), br, (stride, 1), (pad, 0), (dil, 1), G)
        res = None
        if use_res:
            res = torch.randn(y.shape, generator=g)
            resr = res.clone().requires_grad_(True)
            y = y + resr
        if act == 1:
            y = F.leaky_relu(y, 0.1)
        elif act == 2:
            y = torch.relu(y)
        elif act == 3:
            y = torch.tanh(y)
        if masks:
            mo = (torch.arange(y.shape[2])[None, :] < lens[:, None]).float().unsqueeze(1)
            y = y * mo
        gy = torch.randn(y.shape, generator=g)
        y.backward(gy)
        # ---- ours
        to_cl = (lambda t: t.flatten(2).transpose(1, 2).contiguous().to(DEV))
        xd = to_cl(x).requires_grad_(True)
        vd, gd, bd = v.to(DEV).requires_grad_(True), gg.to(DEV).requires_grad_(True), bias.to(DEV).requires_grad_(True)
        # 1-channel inputs / outputs are carried with 4 channels, as models.py does
        pw = ops.pack_weight(vd, gd, pad0=4 if N == 1 else 0, pad1=4 if C == 1 else 0)
        ln = lens.to(DEV).to(torch.int32) if masks else None
        resd = to_cl(res).requires_grad_(True) if use_res else None
        bpad = torch.nn.functional.pad(bd, (0, 3)) if N == 1 else bd
        yo = ops.conv(ops.pad_channels(xd, 4) if C == 1 else xd, pw, bpad, stride=stride, pad=pad, dil=dil, P=P, groups=G,
                      act=act, slope=0.1, res=resd, in_len=ln, out_len=ln)
        if N == 1:
            yo = ops.take_channels(yo, 1)
        yo.backward(to_cl(gy))
        tol = tol_dx = TOL_TC          # every layer (grouped, 1-channel, 1-output) runs on the tensor-core kernels
        # gradients THROUGH a (leaky-)ReLU are compared across different forward roundings: pre-activations within
        # rounding distance of 0 flip their derivative (0.1 <-> 1), which shows up as O(sqrt(flip rate)) relative
        # error (measured 1.0e-2 .. 1.7e-2 in TF32 mode, < 3e-3 in 3xTF32 mode); see test_precise_mode_tightens_conv
        if act in (1, 2) and not PRECISE_MODE[0]:
            tol = tol_dx = max(tol, KINK_TOL)
        elif act in (1, 2):
            tol = tol_dx = max(tol, 5e-3)
        from_cl = lambda t, ref: t.detach().transpose(1, 2).reshape(ref.shape).cpu()
        out.append((f"conv[{name}] y", rel(from_cl(yo, y), y), tol))
        out.append((f"conv[{name}] dx", rel(from_cl(xd.grad, x), xr.grad), tol_dx))
        out.append((f"conv[{name}] dv", rel(vd.grad.cpu(), vr.grad), tol * 2))
        out.append((f"conv[{name}] dg", rel(gd.grad.cpu(), gr.grad), tol * 2))
        out.append((f"conv[{name}] dbias", rel(bd.grad.cpu(), br.grad), tol))
        if use_res:
            out.append((f"conv[{name}] dres", rel(from_cl(resd.grad, res), resr.grad), tol))
    return out


def check_conv_transpose():
    from easevoice_trainer_b200 import ops
    out = []
    for i, (cin, cout, k, s, T) in enumerate([(512, 256, 16, 10, 32), (256, 128, 16, 8, 57), (128, 64, 8, 2, 130),
                                               (64, 32, 2, 2, 300), (32, 16, 2, 2, 500),
                                               (256, 128, 16, 8, 1100), (64, 32, 4, 2, 1500)]):   # large: TMA kernel, os/o0 epilogue
        g = _gen(200 + i)
        x = torch.randn(2, cin, T, generator=g)
        v = torch.randn(cin, cout, k, generator=g) * 0.05
        gg = 0.5 + torch.rand(cin, 1, 1, generator=g)
        b = torch.randn(cout, generator=g) * 0.1
        xr, vr, gr, br = [t.clone().requires_grad_(True) for t in (x, v, gg, b)]
        w = vr * (gr / vr.flatten(1).norm(dim=1).view(-1, 1, 1))
        y = F.conv_transpose1d(xr, w, br, stride=s, padding=(k - s) // 2)
        gy = torch.randn(y.shape, generator=g)
        y.backward(gy)
        xd = cl(x).requires_grad_(True)
        vd, gd, bd = v.to(DEV).requires_grad_(True), gg.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
        yo = ops.conv_transpose(xd, ops.pack_weight(vd, gd), bd, stride=s, pad=(k - s) // 2)
        yo.backward(cl(gy))
        n = f"convT[{cin}->{cout} k{k} s{s}]"
        out += [(n + " y", rel(cf(yo), y), TOL_TC), (n + " dx", rel(cf(xd.grad), xr.grad), TOL_TC),
                (n + " dv", rel(vd.grad.cpu(), vr.grad), TOL_TC2), (n + " dg", rel(gd.grad.cpu(), gr.grad), TOL_TC2),
                (n + " dbias", rel(bd.grad.cpu(), br.grad), TOL_TC)]
    return out


def check_elementwise():
    from easevoice_trainer_b200 import ops
    out = []
    g = _gen(7)
    B, T, C = 3, 37, 48
    lens = torch.tensor([37, 20, 5])
    ln = lens.to(DEV).to(torch.int32)
    mask = (torch.arange(T)[None, :] < lens[:, None]).float().unsqueeze(-1)      # [B,T,1]

    def run(name, fn_ref, fn_ours, inputs, tol=TOL_F32):
        refs = [t.clone().requires_grad_(True) for t in inputs]
        ours = [t.clone().to(DEV).requires_grad_(True) for t in inputs]
        yr = fn_ref(*refs)
        yo = fn_ours(*ours)
        gy = torch.randn(yr.shape, generator=g)
        yr.backward(gy)
        yo.backward(gy.to(DEV))
        out.append((f"ew[{name}] y", rel(yo, yr), tol))
        for k, (a, b) in enumerate(zip(ours, refs)):
            out.append((f"ew[{name}] d{k}", rel(a.grad, b.grad), tol))

    x = torch.randn(B, T, C, generator=g)
    y2 = torch.randn(B, T, C, generator=g)
    y3 = torch.randn(B, T, C, generator=g)
    run("lrelu", lambda a: F.leaky_relu(a, 0.1), lambda a: ops.lrelu(a, 0.1), [x])
    run("tanh", torch.tanh, ops.tanh, [x])
    run("mish", s2_oracle.mish, ops.mish, [x])
    run("add+mask", lambda a, b: (a + b) * mask, lambda a, b: ops.add(a, b, length=ln), [x, y2])
    run("add3", lambda a, b, c: (a + b + c) / 3, lambda a, b, c: ops.add3(a, b, c, 1 / 3, 1 / 3, 1 / 3), [x, y2, y3])
    bv = torch.randn(B, 1, C, generator=g)
    run("add_bvec", lambda a, v: a + v, ops.add_bvec, [x, bv])
    a2 = torch.randn(B, T, 2 * C, generator=g)
    g2 = torch.randn(B, 1, 2 * C, generator=g)
    H = C

    def gate_ref(a, gg):
        t = a + gg
        return torch.tanh(t[..., :H]) * torch.sigmoid(t[..., H:])
    run("wn_gate", gate_ref, ops.wn_gate, [a2, g2])
    run("glu_res", lambda xx, h: xx + h[..., :C] * torch.sigmoid(h[..., C:]), ops.glu_res, [x, a2])
    noise = torch.randn(B, T, C, generator=g)
    run("reparam", lambda st: (st[..., :C] + noise * torch.exp(st[..., C:])) * mask,
        lambda st: ops.reparam(st, noise.to(DEV), ln), [a2 * 0.3])
    run("cat_flip", lambda a, b: torch.cat([a, b], -1).flip(-1), ops.cat_flip, [x, y2])
    ids = torch.tensor([3, 0, 1])
    run("slice_rows", lambda a: torch.stack([a[i, ids[i]:ids[i] + 4] for i in range(B)]),
        lambda a: ops.slice_rows(a, ids.to(DEV), 4), [x])
    w1 = torch.randn(B, 41, 1, generator=g)
    run("reflect_pad", lambda a: F.pad(a.transpose(1, 2), (0, 3), "reflect").transpose(1, 2),
        lambda a: ops.reflect_pad_right(a, 44), [w1])
    tab = torch.randn(20, C, generator=g)
    idx = torch.randint(0, 20, (B, T), generator=g)
    run("embedding", lambda t: F.embedding(idx, t), lambda t: ops.embedding(t, idx.to(DEV)), [tab])
    out.append(("ew[embedding rep2] y", rel(ops.embedding(tab.to(DEV), idx.to(DEV), rep=2),
                                            F.embedding(idx, tab).repeat_interleave(2, dim=1)), 0.0 + 1e-12))
    run("masked_mean", lambda a: (a * mask).sum(1) / lens[:, None].float(), lambda a: ops.masked_mean(a, ln), [x])
    gam, bet = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    run("layernorm", lambda a, r, ga, be: F.layer_norm(a + r, (C,), ga, be, 1e-5),
        lambda a, r, ga, be: ops.layernorm(a, ga, be, res=r), [x, y2, gam, bet], tol=1e-4)
    # layout helpers
    xc = torch.randn(2, 37, 53, generator=g)
    out.append(("ew[to_channels_last]", rel(ops.to_channels_last(xc.to(DEV), pad_to=4), xc.transpose(1, 2)), 1e-12))
    out.append(("ew[to_channels_first]", rel(ops.to_channels_first(xc.to(DEV)), xc.transpose(1, 2)), 1e-12))
    # dropout: keep-rate, scaling, and fwd/bwd mask consistency
    ops.manual_seed(99)
    big = torch.ones(1 << 20, device=DEV, requires_grad=True)
    d = ops.dropout(big, 0.1, "chk")
    d.sum().backward()
    keep = float((d > 0).float().mean())
    out.append(("ew[dropout keep-rate]", abs(keep - 0.9), 3e-3))
    out.append(("ew[dropout scale]", abs(float(d.max()) - 1 / 0.9), 1e-6))
    out.append(("ew[dropout bwd mask == fwd mask]", float((big.grad != d.detach()).float().sum()), 0.5))
    r = ops.randn((1 << 20,), "chk2")
    out.append(("ew[randn mean]", abs(float(r.mean())), 5e-3))
    out.append(("ew[randn std]", abs(float(r.std()) - 1.0), 5e-3))
    return out


def check_attention():
    """Oracle-level relative-L2 row of the parity table; the element-wise gate of the same operator, with the kernel family
    of each contraction asserted, lives in tests/test_gpu_s2_attention_elementwise.py."""
    from easevoice_trainer_b200 import ops
    out = []
    for name, B, Tq, Tk, C, H, win, fill in [("self relpos", 2, 45, 45, 192, 2, 4, -1e4), ("cross", 2, 45, 18, 512, 4, None, -1e4),
                                               ("short relpos T=3", 2, 3, 3, 64, 2, 4, -1e4)]:
        g = _gen(300 + len(name))
        dk = C // H
        q = torch.randn(B, C, Tq, generator=g)
        k = torch.randn(B, C, Tk, generator=g)
        v = torch.randn(B, C, Tk, generator=g)
        ql = torch.tensor([Tq, max(Tq - 9, 1)])
        kl = torch.tensor([Tk, max(Tk - 5, 1)]) if win is None else ql
        P = {"a.conv_q.weight": torch.eye(C).unsqueeze(-1), "a.conv_k.weight": torch.eye(C).unsqueeze(-1),
             "a.conv_v.weight": torch.eye(C).unsqueeze(-1), "a.conv_o.weight": torch.eye(C).unsqueeze(-1)}
        Ek = Ev = None
        if win is not None:
            Ek = (torch.randn(1, 2 * win + 1, dk, generator=g) * dk ** -0.5)
            Ev = (torch.randn(1, 2 * win + 1, dk, generator=g) * dk ** -0.5)
        leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
        if win is not None:
            P["a.emb_rel_k"] = Ek.clone().requires_grad_(True)
            P["a.emb_rel_v"] = Ev.clone().requires_grad_(True)
        qm = (torch.arange(Tq)[None, :] < ql[:, None]).float().unsqueeze(1)
        km = (torch.arange(Tk)[None, :] < kl[:, None]).float().unsqueeze(1)
        am = km.unsqueeze(2) * qm.unsqueeze(-1)
        # the oracle projects q from x and k, v from c; with identity q/k/o projections and a fixed random value
        # projection Wv it computes attention(q=x, k=c, v=Wv c)
        P2 = dict(P)
        Wv = torch.randn(C, C, generator=g) / math.sqrt(C)
        P2["a.conv_v.weight"] = Wv.unsqueeze(-1)
        yr = s2_oracle.relpos_attention(P2, "a", leaves[0], leaves[1], am, H, win)
        gy = torch.randn(yr.shape, generator=g)
        (yr * qm).backward(gy)
        qd, kd = cl(q).requires_grad_(True), cl(k).requires_grad_(True)
        Wvd = Wv.to(DEV)
        vd = torch.matmul(kd, Wvd.t())                 # value path (plain torch matmul only builds the test input)
        Ekd = Ek.to(DEV).requires_grad_(True) if win is not None else None
        Evd = Ev.to(DEV).requires_grad_(True) if win is not None else None
        yo = ops.attention(qd, kd, vd, heads=H, scale=1 / math.sqrt(dk), Ek=Ekd, Ev=Evd, window=win, fill=fill,
                           qlen=ql.to(DEV).to(torch.int32), klen=kl.to(DEV).to(torch.int32))
        qmd = cl(qm)
        (yo * qmd).backward(cl(gy))
        n = f"attn[{name}]"
        out += [(n + " y", rel(cf(yo * qmd), yr * qm), TOL_TC), (n + " dq", rel(cf(qd.grad), leaves[0].grad), TOL_TC2),
                (n + " dk(+v path)", rel(cf(kd.grad), leaves[1].grad), TOL_TC2)]
        if win is not None:
            out += [(n + " dEk", rel(Ekd.grad, P["a.emb_rel_k"].grad), TOL_TC2),
                    (n + " dEv", rel(Evd.grad, P["a.emb_rel_v"].grad), TOL_TC2)]
    return out


def check_vq_losses_optim():
    from easevoice_trainer_b200 import ops
    out = []
    g = _gen(11)
    x = torch.randn(2, 100, 768, generator=g)
    emb = torch.randn(1024, 768, generator=g)
    codes = ops.vq_nearest(x.to(DEV), emb.to(DEV)).cpu()
    ref = s2_oracle.vq_nearest(x.reshape(-1, 768), emb).view(2, 100)
    # bit-exact wherever the fp32 answer is numerically determined (top-2 margin above fp32 rounding of the distance)
    e = emb.t()
    dist = -(x.reshape(-1, 768).pow(2).sum(1, keepdim=True) - 2 * x.reshape(-1, 768) @ e + e.pow(2).sum(0, keepdim=True))
    top2 = dist.topk(2, dim=1).values
    determined = ((top2[:, 0] - top2[:, 1]) > 1e-3).view(2, 100)
    out.append(("vq codes mismatches (determined rows)", float(((codes != ref) & determined).sum()), 0.5))
    out.append(("vq codes mismatches (all rows)", float((codes != ref).sum()), 2.5))
    a = torch.randn(3, 50, 7, generator=g)
    b = torch.randn(3, 50, 7, generator=g)
    for name, fr, fo in [("(1-a)^2", lambda t: torch.mean((1 - t) ** 2), ops.mean_sq_one_minus),
                         ("a^2", lambda t: torch.mean(t ** 2), ops.mean_sq),
                         ("|a-b|", lambda t: torch.mean(torch.abs(b - t)), lambda t: ops.mean_abs_diff(t, b.to(DEV)))]:
        ar = a.clone().requires_grad_(True)
        ao = a.clone().to(DEV).requires_grad_(True)
        lr_, lo = fr(ar), fo(ao)
        (lr_ * 3).backward()
        (lo * 3).backward()
        out += [(f"loss[{name}] value", abs(float(lo) - float(lr_)) / abs(float(lr_)), TOL_F32),
                (f"loss[{name}] grad", rel(ao.grad, ar.grad), TOL_F32)]
    B, T, C = 3, 40, 16
    lens = torch.tensor([40, 22, 9])
    zs = [torch.randn(B, C, T, generator=g) * 0.5 for _ in range(4)]
    refs = [t.clone().requires_grad_(True) for t in zs]
    mask = (torch.arange(T)[None, :] < lens[:, None]).float().unsqueeze(1)
    lr_ = s2_oracle.kl_loss(refs[0], refs[1], refs[2], refs[3], mask)
    lr_.backward()
    ours = [cl(t).requires_grad_(True) for t in zs]
    lo = ops.kl_loss(ours[0], ours[1], ours[2], ours[3], lens.to(DEV).to(torch.int32))
    lo.backward()
    out.append(("loss[kl] value", abs(float(lo) - float(lr_)) / abs(float(lr_)), TOL_F32))
    for i, nm in enumerate(("z_p", "logs_q", "m_p", "logs_p")):
        out.append((f"loss[kl] d{nm}", rel(cf(ours[i].grad), refs[i].grad), TOL_F32))
    # AdamW
    p = torch.randn(10000, generator=g)
    gr = torch.randn(10000, generator=g)
    m = torch.zeros(10000)
    v = torch.zeros(10000)
    pd, gd, md, vd = p.to(DEV), gr.to(DEV), m.to(DEV), v.to(DEV)
    gn = torch.zeros(1, device=DEV)
    hyper = torch.tensor([1e-4, 0.0], device=DEV)
    for step in (1, 2, 3):
        p, m, v = s2_oracle.adamw_step(p, gr, m, v, step, 1e-4)
        ops.scalar_add(hyper[1:], 1.0)
        ops.adamw_flat(pd, gd, md, vd, hyper, 1.0, (0.8, 0.99), 1e-9, 0.01, 1.0, gn)
    out += [("adamw p", rel(pd, p), TOL_F32), ("adamw m", rel(md, m), TOL_F32), ("adamw v", rel(vd, v), TOL_F32),
            ("adamw gnorm", abs(float(gn) / 3 - float((gr ** 2).sum())) / float((gr ** 2).sum()), 1e-5)]
    return out


def check_mel():
    from easevoice_trainer_b200 import mel_processing as mp
    out = []
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "mel_kat_22050.pt"))
    y = mel_oracle.kat_sines()
    mel = mp.mel_spectrogram_torch(y.to(DEV), 2048, 128, 22050, 640, 2048, 0.0, None).cpu()
    spec = mp.spectrogram_torch(y.to(DEV), 2048, 22050, 640, 2048).cpu()
    f64 = torch.from_numpy(mel_oracle.mel_spectrogram_f64(y.numpy(), 2048, 128, 22050, 640, 2048, 0.0, None)).float()
    ref_err = float((gold["mel"] - f64).abs().max())
    # On the pure-tone KAT the fp32 reference itself is 1.2e-3 away from the float64 truth at the spectral floor
    # (bins ~1e-7 of the peak); the kernel must (a) match the reference to 2e-4 wherever the bin is above the floor
    # and (b) be no further from the truth than the reference is.
    floor = f64 < math.log(1e-2)     # mel energy below 1e-2: leakage/rounding-dominated bins of the pure tones
    out.append(("mel KAT |dlogmel| above floor vs reference", float((mel - gold["mel"])[~floor].abs().max()), 2e-4))
    out.append(("mel KAT |dlogmel| vs float64 truth", float((mel - f64).abs().max()), max(2e-4, 1.5 * ref_err)))
    out.append(("mel KAT spec rel-inf vs reference", float(((spec[0] - gold["spec_b0"]).abs() / gold["spec_b0"].abs().clamp(min=1.0)).max()), 1e-3))
    out.append(("mel KAT argmax bins", float((mel[:, :, 17].argmax(1) != torch.tensor([8, 16, 25, 33, 41, 48, 54, 59])).sum()), 0.5))
    for sr, L in ((32000, 32000), (48000, 24000)):
        gd = torch.load(os.path.join(ROOT, "tests", "golden", f"mel_rand_{sr}.pt"))
        g = _gen(7)
        ys = [torch.rand(3, LL, generator=g) - 0.5 for LL in (32000, 24000)]
        yy = ys[0] if sr == 32000 else ys[1]
        m = mp.mel_spectrogram_torch(yy.to(DEV), 2048, 128, sr, 640, 2048, 0.0, None).cpu()
        out.append((f"mel random audio sr={sr} |dlogmel| vs reference golden", float((m - gd["mel"]).abs().max()), 2e-4))
        sp = mp.spectrogram_torch(yy.to(DEV), 2048, sr, 640, 2048)
        m2 = mp.spec_to_mel_torch(sp, 2048, 128, sr, 0.0, None).cpu()
        out.append((f"spec_to_mel(spectrogram) == mel sr={sr}", float((m2 - m).abs().max()), 1e-5))
    # backward
    g = _gen(3)
    yy = (torch.rand(2, 20480, generator=g) - 0.5)
    yr = yy.clone().requires_grad_(True)
    mr = mel_oracle.mel_spectrogram(yr, 2048, 128, 32000, 640, 2048, 0.0, None)
    gy = torch.randn(mr.shape, generator=g)
    mr.backward(gy)
    yo = yy.clone().to(DEV).requires_grad_(True)
    mo = mp.mel_spectrogram_torch(yo, 2048, 128, 32000, 640, 2048, 0.0, None)
    mo.backward(gy.to(DEV))
    out.append(("mel backward d wav", rel(yo.grad, yr.grad), 1e-4))
    return out


def check_stft():
    """General STFT kernel + adjoint (stft.cu) vs torch.stft on the CPU: every (n_fft, hop, win) of the MR-STFT loss, the
    per-row-length front end, the block-per-frame variant of the training configuration, and the MR-STFT loss with its gradient."""
    from easevoice_trainer_b200 import ops, lib
    from easevoice_trainer_b200 import mel_processing as mp
    out = []
    g = _gen(21)
    y = torch.rand(3, 6000, generator=g) - 0.5
    for n_fft, hop, win, center in ((2048, 147, 2048, True), (4096, 147, 4096, True), (2048, 147, 1024, True), (2048, 147, 512, True),
                                    (2048, 147, 256, True), (1024, 256, 1024, True), (512, 128, 512, False), (256, 64, 256, True)):
        yr = y.clone().requires_grad_(True)
        ref = torch.view_as_real(torch.stft(yr, n_fft, hop_length=hop, win_length=win, window=torch.hann_window(win), center=center,
                                            pad_mode="reflect", normalized=False, onesided=True, return_complex=True)).permute(0, 2, 1, 3)
        gy = torch.randn(ref.shape, generator=g)
        (ref * gy).sum().backward()
        yd = y.to(DEV).requires_grad_(True)
        o = ops.stft(yd, n_fft, hop, win, center=center)
        (o * gy.to(DEV)).sum().backward()
        tag = f"stft n_fft={n_fft} hop={hop} win={win} center={center}"
        out.append((tag + " X", rel(o, ref), 2e-6))
        out.append((tag + " d wav (adjoint)", rel(yd.grad, yr.grad), 5e-6))
    # MR-STFT loss of bs_roformer.py:565-581 (complex L1 over five windows) and its gradient
    yh = (torch.rand(2, 12000, generator=g) - 0.5)
    yt = (torch.rand(2, 12000, generator=g) - 0.5)
    yhr = yh.clone().requires_grad_(True)
    tot = 0
    for w in (4096, 2048, 1024, 512, 256):
        kw = dict(n_fft=max(w, 2048), hop_length=147, win_length=w, window=torch.hann_window(w), return_complex=True, normalized=False)
        tot = tot + F.l1_loss(torch.stft(yhr, **kw), torch.stft(yt, **kw))
    tot.backward()
    yhd = yh.to(DEV).requires_grad_(True)
    lo = ops.mrstft_loss(yhd, yt.to(DEV))
    lo.backward()
    out.append(("mrstft loss", abs(float(lo) - float(tot)) / float(tot), 1e-5))
    out.append(("mrstft d y_hat", rel(yhd.grad, yhr.grad), 2e-5))
    # per-row lengths: |X| of a zero-padded batch == the reference's per-utterance spectrogram + zero-padding collate
    L = 640 * 40
    wav = torch.zeros(3, L)
    lens = [L, 640 * 33 + 17, 640 * 21]
    for b, n in enumerate(lens):
        wav[b, :n] = torch.rand(n, generator=g) - 0.5
    ref = torch.zeros(3, 1025, 40)
    for b, n in enumerate(lens):
        sp = mel_oracle.spectrogram(wav[b:b + 1, :n], 2048, 640, 2048)
        ref[b, :, :sp.shape[2]] = sp[0]
    ln = torch.tensor(lens, dtype=torch.int32, device=DEV)
    got = mp.spectrogram_torch(wav.to(DEV), 2048, 32000, 640, 2048, lengths=ln)
    out.append(("spectrogram with per-row lengths (warp kernel)", rel(got, ref), 2e-5))
    L_ = lib.init()
    L_.evk_set_mel_variant(0)
    try:
        got0 = mp.spectrogram_torch(wav.to(DEV), 2048, 32000, 640, 2048, lengths=ln)
        m0 = mp.mel_spectrogram_torch(wav.to(DEV), 2048, 128, 32000, 640, 2048, 0.0, None)
    finally:
        L_.evk_set_mel_variant(1)
    m1 = mp.mel_spectrogram_torch(wav.to(DEV), 2048, 128, 32000, 640, 2048, 0.0, None)
    out.append(("spectrogram with per-row lengths (general kernel)", rel(got0, ref), 2e-5))
    out.append(("log-mel: general kernel vs warp kernel, max |d|", float((m0 - m1).abs().max()), 2e-4))
    # a non-default transform size through the reference-named API (n_fft 1024 / win 512 / hop 160)
    y2 = torch.rand(2, 8000, generator=g) - 0.5
    ref2 = mel_oracle.spectrogram(y2, 1024, 160, 512)
    out.append(("spectrogram_torch n_fft=1024 hop=160 win=512", rel(mp.spectrogram_torch(y2.to(DEV), 1024, 32000, 160, 512), ref2), 2e-5))
    return out


def check_fused_dropout():
    """Dropout fused into the GEMM epilogue (linear + ReLU + dropout, backward from the saved output) and into LayerNorm
    (LN(x + dropout(res)), mask regenerated in the backward): the mask is recovered from the kernels' own outputs and the
    results are compared with the unfused operators applied with that mask."""
    from easevoice_trainer_b200 import ops
    out = []
    g = _gen(77)
    p = 0.1
    # ---- linear -> ReLU -> dropout
    x = torch.randn(4, 256, 128, generator=g).to(DEV)
    v = (torch.randn(256, 128, 1, generator=g) * 0.1).to(DEV)
    b = (torch.randn(256, generator=g) * 0.1).to(DEV)
    gy = torch.randn(4, 256, 256, generator=g).to(DEV)
    xa, va, ba = [t.clone().requires_grad_(True) for t in (x, v, b)]
    pw = ops.pack_weight(va, None)
    ops.dispatch_reset()
    yf = ops.linear(xa, pw, ba, act=ops.ACT_RELU, drop=(p, "chk.drop.lin"))
    # TF32 mode: the dropout is fused into gemm_tma_kernel's epilogue; 3xTF32 mode runs mma.sync and then the dropout pass
    want = "fwd_mma_sync" if PRECISE_MODE[0] else "fwd_gemm_tma"
    disp = ops.dispatch_stats()
    served = disp[want] > 0 and not any(disp[k] for k in ops.DISPATCH_SLOTS if k.startswith("fwd_") and k != want)
    out.append((f"linear + ReLU + dropout served by {want}", 0.0 if served else 1.0, 0.5))
    yf.backward(gy)
    xb, vb, bb = [t.clone().requires_grad_(True) for t in (x, v, b)]
    yp = ops.linear(xb, ops.pack_weight(vb, None), bb, act=ops.ACT_RELU)
    pos = yp.detach() > 0
    M = ((yf.detach() != 0) & pos).float() / (1.0 - p)
    out.append(("linear+relu+dropout: kept values = relu(.)/(1-p), dropped = 0", rel(yf, yp.detach() * M), 1e-6))
    frac = 1.0 - float(((yf.detach() != 0) & pos).sum()) / float(pos.sum())
    out.append(("linear+relu+dropout: drop fraction vs p", abs(frac - p) / p, 5e-2))
    (yp * M).backward(gy)
    out.append(("linear+relu+dropout dx (mask-free backward from the saved output)", rel(xa.grad, xb.grad), TOL_TC2))
    out.append(("linear+relu+dropout dW", rel(va.grad, vb.grad), TOL_TC2))
    out.append(("linear+relu+dropout dbias", rel(ba.grad, bb.grad), 1e-5))
    # ---- LayerNorm(x + dropout(res))
    x = torch.randn(4, 300, 512, generator=g).to(DEV)
    a = torch.randn(4, 300, 512, generator=g).to(DEV)
    gm = (1.0 + 0.1 * torch.randn(512, generator=g)).to(DEV)
    bt = (0.1 * torch.randn(512, generator=g)).to(DEV)
    gy = torch.randn(4, 300, 512, generator=g).to(DEV)
    x1, a1, g1, b1 = [t.clone().requires_grad_(True) for t in (x, a, gm, bt)]
    y1 = ops.layernorm(x1, g1, b1, res=a1, res_drop=(p, "chk.drop.ln"))
    y1.backward(gy)
    ratio = a1.grad / x1.grad                                   # = mask / (1-p) wherever dx != 0
    M = (ratio.abs() > 0.5).float() / (1.0 - p)
    out.append(("LN+dropout: dres = dx * mask/(1-p) (mask is 0/1)", float((ratio - M).abs().max()), 1e-5))
    out.append(("LN+dropout: drop fraction vs p", abs(float((M == 0).float().mean()) - p) / p, 5e-2))
    x2, a2, g2, b2 = [t.clone().requires_grad_(True) for t in (x, a, gm, bt)]
    y2 = ops.layernorm(x2, g2, b2, res=a2 * M)
    y2.backward(gy)
    out.append(("LN+dropout forward vs unfused LN(x + res * mask/(1-p))", rel(y1, y2), 2e-6))
    out.append(("LN+dropout dx", rel(x1.grad, x2.grad), 2e-5))
    out.append(("LN+dropout dres", rel(a1.grad, a2.grad), 2e-5))
    out.append(("LN+dropout dgamma", rel(g1.grad, g2.grad), 2e-5))
    out.append(("LN+dropout dbeta", rel(b1.grad, b2.grad), 2e-5))
    # gamma / beta as 4-byte-aligned views of flat parameter storage (the DPO trainer's layout)
    flat = torch.zeros(2 * 512 + 3, device=DEV)
    flat[1:513] = gm; flat[514:1026] = bt
    y3 = ops.layernorm(x, flat[1:513], flat[514:1026], res=a, res_drop=(p, "chk.drop.ln"))
    out.append(("LN+dropout with gamma/beta at odd element offsets == aligned result", rel(y3, y1.detach()), 0.0))
    return out


def _load_models(seed_g=1234, seed_d=4321):
    from easevoice_trainer_b200 import models
    net_g = models.SynthesizerTrn(1025, 32, n_speakers=300, **s2_oracle.S2_MODEL)
    net_d = models.MultiPeriodDiscriminator(False)
    PG = s2_oracle.init_params(s2_oracle.generator_param_spec(), seed_g)
    PD = s2_oracle.init_params(s2_oracle.discriminator_param_spec(), seed_d)
    net_g.load_state_dict(PG)
    net_d.load_state_dict(PD)
    return net_g.to(DEV).eval(), net_d.to(DEV).eval(), PG, PD


def check_s2(tag="small"):
    """Assembled networks + both losses + parameter gradients vs the oracle, and vs the committed reference goldens."""
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.train import s2_step
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", f"s2_{tag}.json")))
    c = gold["cfg"]
    B, T, X = c["B"], c["T"], c["X"]
    net_g, net_d, PG, PD = _load_models(c["g_seed"], c["d_seed"])
    wav, ssl, text, spec_len, text_len = s2_oracle.synthetic_batch(B, T, X, c["batch_seed"], c["ragged"])
    spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, 640, 2048)
    g = _gen(c["noise_seed"])
    noise = torch.randn(B, 192, T, generator=g)
    ids = (torch.rand(B, generator=g) * (spec_len - 32 + 1)).long()
    assert ids.tolist() == gold["ids_slice"]
    # oracle
    OG = {k: (v.clone().requires_grad_(True) if k not in s2_oracle.GEN_BUFFERS else v.clone()) for k, v in PG.items()}
    OD = {k: v.clone().requires_grad_(True) for k, v in PD.items()}
    o = s2_oracle.s2_losses(OG, OD, (ssl, spec, spec_len, wav, text, text_len), noise, ids)
    for k in ("loss_disc", "loss_gen_all"):
        out.append((f"s2[{tag}] oracle {k} vs reference golden", abs(float(o[k]) - gold[k]) / abs(gold[k]), 1e-4))
    gd_ref = dict(zip(OD.keys(), torch.autograd.grad(o["loss_disc"], list(OD.values()), retain_graph=True)))
    gn = [k for k in OG if k not in s2_oracle.GEN_BUFFERS]
    gg_ref = dict(zip(gn, torch.autograd.grad(o["loss_gen_all"], [OG[k] for k in gn], allow_unused=True)))
    # ours
    hps_t = dict(s2_oracle.S2_TRAIN)
    hps_d = dict(s2_oracle.S2_DATA)
    stepper = s2_step.S2Step(net_g, net_d, hps_t, hps_d)
    batch = dict(ssl=cl(ssl), spec=ops.to_channels_last(spec.to(DEV), pad_to=4), lengths=spec_len.to(DEV).to(torch.int32),
                 wav=wav.reshape(B, -1, 1).to(DEV), text=text.to(DEV), text_lengths=text_len.to(DEV).to(torch.int32))
    r = stepper.losses(batch, noise=cl(noise), ids_slice=ids.to(DEV))
    out.append((f"s2[{tag}] VQ codes mismatches", float((r["codes"].cpu() != o["codes"]).sum()), 0.5))
    for k in ("z", "z_p", "m_p", "logs_p", "m_q", "logs_q", "y_hat"):
        out.append((f"s2[{tag}] {k}", rel(cf(r[k]), o[k]), TOL_NET))
    out.append((f"s2[{tag}] y_hat_mel", rel(cf(r["y_hat_mel"]), o["y_hat_mel"]), TOL_NET))
    out.append((f"s2[{tag}] y_mel", rel(cf(r["y_mel"]), o["y_mel"]), 1e-5))
    out.append((f"s2[{tag}] y slice", rel(cf(r["y"]), o["y"]), 1e-12))
    ld = stepper.d_loss(r)
    lg, parts = stepper.g_loss(r)
    out.append((f"s2[{tag}] loss_disc", abs(float(ld) - float(o["loss_disc"])) / float(o["loss_disc"]), TOL_NET))
    out.append((f"s2[{tag}] loss_gen_all", abs(float(lg) - float(o["loss_gen_all"])) / float(o["loss_gen_all"]), TOL_NET))
    for k in ("loss_gen", "loss_fm", "loss_mel", "loss_kl"):
        out.append((f"s2[{tag}] {k}", abs(float(parts[k]) - float(o[k])) / abs(float(o[k])), TOL_NET))
        out.append((f"s2[{tag}] {k} vs reference golden", abs(float(parts[k]) - gold[k]) / abs(gold[k]), TOL_NET))
    dnames = [n for n, _ in net_d.named_parameters()]
    gd = torch.autograd.grad(ld, [p for _, p in net_d.named_parameters()], retain_graph=True, allow_unused=True)
    worst, wname, num, den = 0.0, "", 0.0, 0.0
    for n, gr in zip(dnames, gd):
        e = rel(gr, gd_ref[n])
        num += float((gr.detach().double().cpu() - gd_ref[n].double()).pow(2).sum())
        den += float(gd_ref[n].double().pow(2).sum())
        if e > worst:
            worst, wname = e, n
    # per-tensor worst case is dominated by leaky-ReLU derivative flips in the 1->32 / 1->16 first layers (KINK_TOL x2)
    out.append((f"s2[{tag}] D param grads worst rel-L2 ({wname})", worst, NET_GRAD_TENSOR))
    out.append((f"s2[{tag}] D param grads global rel-L2", math.sqrt(num / den), NET_GRAD_GLOBAL))
    gnames = [n for n, _ in net_g.named_parameters()]
    gg = torch.autograd.grad(lg, [p for _, p in net_g.named_parameters()], allow_unused=True)
    worst, wname, unused = 0.0, "", []
    tot_num, tot_den = 0.0, 0.0
    for n, gr in zip(gnames, gg):
        if gr is None:
            unused.append(n)
            continue
        if n.endswith(("conv_k.bias", "w_ks.bias")):       # analytically zero gradients (see pin_against_reference.py)
            continue
        e = rel(gr, gg_ref[n])
        tot_num += float((gr.detach().double().cpu() - gg_ref[n].double()).pow(2).sum())
        tot_den += float(gg_ref[n].double().pow(2).sum())
        if e > worst:
            worst, wname = e, n
    out.append((f"s2[{tag}] G param grads worst rel-L2 ({wname})", worst, NET_GRAD_TENSOR))
    out.append((f"s2[{tag}] G param grads global rel-L2", math.sqrt(tot_num / tot_den), NET_GRAD_GLOBAL))
    out.append((f"s2[{tag}] unused G params == {{ssl_proj.weight, ssl_proj.bias}}",
                0.0 if sorted(unused) == ["ssl_proj.bias", "ssl_proj.weight"] else 1.0, 0.5))
    for k, v in gold["grad_norms_g"].items():
        gr = gg[gnames.index(k)]
        out.append((f"s2[{tag}] |grad {k}| vs reference golden", abs(float(gr.norm()) - v) / v, 3e-2))
    return out


def check_api_layouts():
    """Reference-contract entry points ([B,C,T] in/out) agree with the channels-last fast path."""
    out = []
    net_g, net_d, PG, PD = _load_models()
    B, T, X = 2, 40, 9
    wav, ssl, text, spec_len, text_len = s2_oracle.synthetic_batch(B, T, X, 5, True)
    spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, 640, 2048)
    g = _gen(1)
    noise = torch.randn(B, 192, T, generator=g)
    ids = torch.tensor([2, 0])
    o = s2_oracle.synthesizer_forward(PG, ssl, spec, spec_len, text, text_len, noise, ids)
    y_hat, commit, ids_r, m1, m2, lat, quant = net_g(ssl.to(DEV), spec.to(DEV), spec_len.to(DEV), text.to(DEV),
                                                     text_len.to(DEV), noise=noise.to(DEV), ids_slice=ids.to(DEV))
    out.append(("api G y_hat [B,1,T]", rel(y_hat, o["y_hat"]), TOL_NET))
    out.append(("api G quantized", rel(quant, o["quantized"]), 1e-12))
    out.append(("api G mask", rel(m1, o["y_mask"]), 1e-12))
    for t, k in zip(lat, ("z", "z_p", "m_p", "logs_p", "m_q", "logs_q")):
        out.append((f"api G {k}", rel(t, o[k]), TOL_NET))
    y = torch.rand(2, 1, 20480, generator=g) - 0.5
    yh = torch.rand(2, 1, 20480, generator=g) - 0.5
    rs, gs, frs, fgs = s2_oracle.mpd(PD, y, yh)
    ors, ogs, ofrs, ofgs = net_d(y.to(DEV), yh.to(DEV))
    for d in range(6):
        out.append((f"api D[{d}] logits real", rel(ors[d], rs[d]), TOL_NET))
        out.append((f"api D[{d}] logits gen", rel(ogs[d], gs[d]), TOL_NET))
        for i in range(len(frs[d])):
            out.append((f"api D[{d}] fmap{i}", rel(ofgs[d][i], fgs[d][i]), TOL_NET))
    return out


# ------------------------------------------------------------------------------------------------
# stage-1 AR GPT
# ------------------------------------------------------------------------------------------------
def _sdpa_oracle(qkv, H, X, xl, yl, keep=None, p=0.0):
    """reference attention core on CPU: mask of t2s_model.py:456-479, softmax, optional given dropout keep-mask."""
    B, L, D3 = qkv.shape
    D = D3 // 3
    dk = D // H
    q, k, v = [t.view(B, L, H, dk).transpose(1, 2) for t in qkv.split(D, dim=-1)]
    mask = gpt_oracle.prefix_lm_mask(xl, yl, X, L - X)
    add = torch.zeros(mask.shape).masked_fill(mask, float("-inf")).unsqueeze(1)
    P = torch.softmax(q @ k.transpose(-2, -1) / math.sqrt(dk) + add, dim=-1)
    if keep is not None:
        P = P * keep / (1.0 - p)
    return (P @ v).transpose(1, 2).reshape(B, L, D)


def check_gpt_kernels():
    from easevoice_trainer_b200 import ops
    out = []
    # ---- fused prefix-LM attention, no dropout: forward + all three gradients, ragged lens, L not a tile multiple
    for tag, B, H, X, Y, seed in (("small", 2, 2, 7, 30, 1), ("tiles", 2, 3, 70, 150, 2), ("x-only-tail", 1, 1, 64, 1, 3)):
        g = _gen(seed)
        L, D = X + Y, H * 32
        qkv = torch.randn(B, L, 3 * D, generator=g)
        xl = torch.randint(max(X // 2, 1), X + 1, (B,), generator=g); xl[0] = X
        yl = torch.randint(max(Y // 2, 1), Y + 1, (B,), generator=g); yl[0] = Y
        go = torch.randn(B, L, D, generator=g)
        qr = qkv.clone().requires_grad_(True)
        o_ref = _sdpa_oracle(qr, H, X, xl, yl)
        o_ref.backward(go)
        qd = qkv.to(DEV).requires_grad_(True)
        o = ops.flash_attention(qd, heads=H, prefix=X, xlen=xl.to(DEV), ylen=yl.to(DEV))
        o.backward(go.to(DEV))
        out.append((f"flash {tag} out", rel(o, o_ref), TOL_TC))
        gq, gk, gv = qd.grad.cpu().split(D, dim=-1)
        rq, rk, rv = qr.grad.split(D, dim=-1)
        out.append((f"flash {tag} dq", rel(gq, rq), TOL_TC2))
        out.append((f"flash {tag} dk", rel(gk, rk), TOL_TC2))
        out.append((f"flash {tag} dv", rel(gv, rv), TOL_TC2))
    # ---- dropout: recover the keep mask with V = I (L = 32 keys, dk = 32), then check fwd/bwd against the oracle given it
    B, H, X, Y, p = 2, 2, 12, 20, 0.25
    L, D = 32, 64
    g = _gen(9)
    ops.manual_seed(77)
    qkv = torch.randn(B, L, 3 * D, generator=g)
    xl, yl = torch.tensor([12, 9]), torch.tensor([20, 13])
    probe = qkv.clone()
    probe[:, :, 2 * D:] = torch.eye(32).repeat(1, H)[None]
    pd = ops.flash_attention(probe.to(DEV), heads=H, prefix=X, xlen=xl.to(DEV), ylen=yl.to(DEV), p_drop=p, tag="chk.drop").cpu()
    pd = pd.view(B, L, H, 32).transpose(1, 2)                                   # [B,H,i,j] = dropped probabilities
    p0 = ops.flash_attention(probe.to(DEV), heads=H, prefix=X, xlen=xl.to(DEV), ylen=yl.to(DEV)).cpu().view(B, L, H, 32).transpose(1, 2)
    vis = p0 > 1e-6
    keep = (pd != 0) | ~vis
    frac = float(((pd == 0) & vis).sum()) / float(vis.sum())
    out.append(("flash dropout drop-fraction vs p", abs(frac - p), 0.05))
    out.append(("flash dropout kept values = P/(1-p)", rel(pd[keep & vis], (p0 / (1 - p))[keep & vis]), TOL_TC))
    go = torch.randn(B, L, D, generator=g)
    qr = qkv.clone().requires_grad_(True)
    o_ref = _sdpa_oracle(qr, H, X, xl, yl, keep.float(), p)
    o_ref.backward(go)
    qd = qkv.to(DEV).requires_grad_(True)
    o = ops.flash_attention(qd, heads=H, prefix=X, xlen=xl.to(DEV), ylen=yl.to(DEV), p_drop=p, tag="chk.drop")
    o.backward(go.to(DEV))
    out.append(("flash dropout out (same mask)", rel(o, o_ref), TOL_TC))
    out.append(("flash dropout dqkv (mask regenerated in bwd)", rel(qd.grad, qr.grad), TOL_TC2))
    # ---- sinusoid + alpha + concat
    from easevoice_trainer_b200.models_gpt import sine_table
    B, X, Y, D = 3, 5, 9, 64
    xe, ye = torch.randn(B, X, D, generator=g), torch.randn(B, Y, D, generator=g)
    ax, ay = torch.tensor([0.7]), torch.tensor([1.4])
    pe = gpt_oracle.sine_pe(16, D)
    out.append(("sine table == oracle", rel(sine_table(16, D), pe), 0.0))
    ins = [t.clone().requires_grad_(True) for t in (xe, ye, ax, ay)]
    ref = torch.cat([ins[0] + ins[2] * pe[:X], ins[1] + ins[3] * pe[:Y]], 1)
    gh = torch.randn(B, X + Y, D, generator=g)
    ref.backward(gh)
    dins = [t.to(DEV).requires_grad_(True) for t in (xe, ye, ax, ay)]
    h = ops.gpt_embed(*dins, pe.to(DEV))
    h.backward(gh.to(DEV))
    out.append(("gpt_embed h", rel(h, ref), TOL_F32))
    for nm, a, b in zip(("dxe", "dye", "dalpha_x", "dalpha_y"), dins, ins):
        out.append((f"gpt_embed {nm}", rel(a.grad, b.grad), TOL_F32))
    # ---- CE(sum) + top-3 accuracy ignoring EOS, padded class dim
    rows, V = 333, 1025
    lg = torch.randn(rows, V, generator=g) * 3
    tg = torch.randint(0, V, (rows,), generator=g); tg[::7] = 1024
    for r in range(0, rows, 3):
        lg[r, tg[r]] += 6.0
    lr_ = lg.clone().requires_grad_(True)
    loss_ref = F.cross_entropy(lr_, tg, reduction="sum")
    (loss_ref * 0.5).backward()
    top3 = lg.topk(3, dim=-1).indices
    valid = tg != 1024
    acc_ref = ((top3 == tg[:, None]).any(-1) & valid).sum().float() / valid.sum().float()
    lp = torch.zeros(rows, 1028); lp[:, :V] = lg
    ld_ = lp.to(DEV).requires_grad_(True)
    loss, out2 = ops.ce_sum_topk(ld_, tg.to(DEV), 3, 1024, V=V)
    (loss * 0.5).backward()
    out.append(("ce loss sum", rel(loss, loss_ref), TOL_F32))
    out.append(("ce top-3 acc (exact count)", abs(float(out2[1]) - float(acc_ref)), 1e-7))
    out.append(("ce dlogits", rel(ld_.grad[:, :V], lr_.grad), TOL_F32))
    out.append(("ce dlogits pad cols zero", float(ld_.grad[:, V:].abs().max()), 0.0))
    return out


def check_scaled_adam():
    """30 steps on the pinned golden trajectory (tests/golden/scaled_adam.json, produced by the reference class)."""
    from easevoice_trainer_b200.train.gpt_step import FlatScaledAdam
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "scaled_adam.json")))
    g = _gen(gold["seed"])
    shapes = [tuple(s) for s in gold["shapes"]]
    init = [torch.randn(s, generator=g) * sc for s, sc in zip(shapes, gold["scales"])]
    po = [t.clone() for t in init]
    oo = gpt_oracle.ScaledAdamOracle(po, lr=gold["lr_first"], clipping_update_period=gold["clipping_update_period"])
    params = [torch.nn.Parameter(t.clone().to(DEV)) for t in init]
    opt = FlatScaledAdam([(f"p{i}", p) for i, p in enumerate(params)], lr=gold["lr_first"],
                         clipping_update_period=gold["clipping_update_period"])
    worst, worst_gold, cs_seen = 0.0, 0.0, 1.0
    for it in range(gold["steps"]):
        grads = [torch.randn(s, generator=g) * (5.0 if it in gold["big_grad_steps"] else 1.0) for s in shapes]
        opt.accumulate([x.to(DEV) for x in grads])
        opt.step()
        cs = oo.step(grads)
        cs_seen = min(cs_seen, float(cs))
        if it == 0:
            opt.set_lr(gold["lr_rest"]); oo.lr = gold["lr_rest"]
        worst = max(worst, max(rel(a.data, b) for a, b in zip(params, po)))
        worst_gold = max(worst_gold, max(abs(float(a.data.double().norm()) - n) / (n + 1e-12) for a, n in zip(params, gold["param_norms"][it])))
    out.append(("scaled_adam 30-step trajectory vs oracle", worst, 2e-5))
    out.append(("scaled_adam 30-step param norms vs reference golden", worst_gold, 2e-5))
    out.append(("scaled_adam clipping engaged (cs < 1 seen)", 0.0 if cs_seen < 1.0 else 1.0, 0.5))
    out.append(("scaled_adam grads zeroed", float(opt.flat_g.abs().max()), 0.0))
    out.append(("scaled_adam step counter", abs(opt.step_count - gold["steps"]), 0))
    return out


def check_gpt(tag="small"):
    """assembled forward_old + backward vs the oracle and the reference golden (dropout off), then 6 training_steps
    (accumulate-4 + ScaledAdam) vs the oracle loop."""
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    from easevoice_trainer_b200.train.gpt_step import GptStep
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", f"gpt_{tag}.json")))
    m = gold["model"]
    spec = gpt_oracle.gpt_param_spec(m)
    P = gpt_oracle.init_params(spec, gold["param_seed"])
    P["ar_text_position.alpha"].fill_(gold["alpha_text"]); P["ar_audio_position.alpha"].fill_(gold["alpha_audio"])
    net = Text2SemanticDecoder({"model": m}, layer_dropout=0.0)
    sd = net.state_dict()
    out.append((f"gpt {tag} state_dict keys/shapes == reference", 0.0 if {k: tuple(v.shape) for k, v in sd.items()} == spec else 1.0, 0.0))
    net.load_state_dict(P)
    net = net.to(DEV)
    x, xl, y, yl, bert = gpt_oracle.synthetic_gpt_batch(gold["B"], gold["X"], gold["Y"], gold["batch_seed"], gold["ragged"])
    Pq = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    taps = {}
    loss_o, acc_o, logits_o, tg_o = gpt_oracle.forward_old(Pq, x, xl, y, yl, bert, m, taps)
    loss_o.backward()
    loss, acc = net.forward_old(x.to(DEV), xl.to(DEV), y.to(DEV), yl.to(DEV), bert.to(DEV))
    names = [n for n, _ in net.named_parameters()]
    grads = torch.autograd.grad(loss, [p for _, p in net.named_parameters()])
    y_in, tg = net.make_targets(y.to(DEV), yl.to(DEV))
    out.append((f"gpt {tag} targets (pad_y_eos) exact", float((tg.cpu() != tg_o).sum()), 0.0))
    out.append((f"gpt {tag} targets checksum == reference golden", abs(int(tg.sum()) - gold["targets_sum"]), 0))
    out.append((f"gpt {tag} logits", rel(net.last_logits[..., :m["vocab_size"]].reshape(logits_o.shape), logits_o), TOL_NET))
    out.append((f"gpt {tag} loss vs oracle", abs(float(loss.detach()) - float(loss_o)) / abs(float(loss_o)), TOL_NET))
    out.append((f"gpt {tag} loss vs reference golden", abs(float(loss.detach()) - gold["loss"]) / abs(gold["loss"]), TOL_NET))
    out.append((f"gpt {tag} top-3 acc vs reference golden", abs(float(acc) - gold["acc"]), 2.0 / (gold["B"] * gold["Y"])))
    worst, gl = 0.0, 0.0
    num = den = 0.0
    # d(alpha) = <dh, pe> projects the whole [B, L, D] gradient onto one direction (heavy cancellation): a relative
    # perturbation eps of dh moves it by ~ eps * |dh| * rms(pe) in ABSOLUTE terms (rms(pe) = 1/sqrt 2), however small the
    # result is.  So alpha is checked against the noise level measured on all the other tensors (4 sigma).
    alpha_rows = []
    for n, gk in zip(names, grads):
        if n.endswith(".alpha"):
            alpha_rows.append((n, abs(float(gk) - float(Pq[n].grad))))
            continue
        r = rel(gk, Pq[n].grad)
        worst = max(worst, r)
        num += float((gk.cpu().double() - Pq[n].grad.double()).pow(2).sum()); den += float(Pq[n].grad.double().pow(2).sum())
        if n in gold["grad_norms"]:
            gl = max(gl, abs(float(gk.norm()) - gold["grad_norms"][n]) / (gold["grad_norms"][n] + 1e-12))
    alpha_tol = 4.0 * max(math.sqrt(num / den), 1e-4) * float(taps["h0"].grad.norm()) * math.sqrt(0.5)
    for n, e in alpha_rows:
        out.append((f"gpt {tag} d{n} (abs, projection-noise bound)", e, alpha_tol))
    out.append((f"gpt {tag} grads worst tensor", worst, 2 * KINK_TOL))
    out.append((f"gpt {tag} grads global", math.sqrt(num / den), KINK_TOL))
    out.append((f"gpt {tag} grad norms vs reference golden", gl, 2e-2))
    if tag == "small":
        # 6 x training_step: update after batch_idx 4 only (5 accumulated micro-batches), lr 0.01 for that first update
        step = GptStep(net)
        Po = [v.detach().clone() for v in Pq.values()]
        keys = list(Pq.keys())
        oo = gpt_oracle.ScaledAdamOracle(Po, lr=0.01)
        acc_g = [torch.zeros_like(v) for v in Po]
        lo = []
        for it in range(6):
            xb, xlb, yb, ylb, bb = gpt_oracle.synthetic_gpt_batch(gold["B"], gold["X"], gold["Y"], 100 + it, it % 2 == 1)
            Pr = {k: v.clone().requires_grad_(True) for k, v in zip(keys, Po)}
            l_o = gpt_oracle.forward_old(Pr, xb, xlb, yb, ylb, bb, m)[0]
            l_o.backward()
            for a, k in zip(acc_g, keys):
                a += Pr[k].grad
            if it > 0 and it % 4 == 0:
                oo.step(acc_g)
                oo.lr = 0.002
                acc_g = [torch.zeros_like(v) for v in Po]
            l_d, _ = step.step(dict(phoneme_ids=xb.to(DEV), phoneme_ids_len=xlb.to(DEV), semantic_ids=yb.to(DEV),
                                    semantic_ids_len=ylb.to(DEV), bert_feature=bb.to(DEV)))
            lo.append(abs(float(l_d) - float(l_o)) / abs(float(l_o)))
        out.append(("gpt 6 training_steps: loss track", max(lo), TOL_NET))
        out.append(("gpt 6 training_steps: exactly one optimizer step", abs(step.opt.step_count - 1), 0))
        pw = max(rel(p.data, Po[keys.index(n)]) for n, p in net.named_parameters())
        out.append(("gpt 6 training_steps: params vs oracle loop", pw, 2e-3))
    return out


def check_gpt_dpo_and_trainer():
    """DPO variant of the step (if_dpo) vs the oracle + reference golden, then GPTTrain end to end on a tiny synthetic
    dataset (files in the reference's layout): stdout protocol, checkpoint layout and resume."""
    import contextlib
    import io
    import tempfile
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder, make_reject_y
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "gpt_ragged.json")))
    m = gold["model"]
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), gold["param_seed"])
    P["ar_text_position.alpha"].fill_(gold["alpha_text"]); P["ar_audio_position.alpha"].fill_(gold["alpha_audio"])
    net = Text2SemanticDecoder({"model": m}, layer_dropout=0.0)
    net.load_state_dict(P)
    net = net.to(DEV)
    x, xl, y, yl, bert = gpt_oracle.synthetic_gpt_batch(gold["B"], gold["X"], gold["Y"], gold["batch_seed"], gold["ragged"])
    ry, ryl = gpt_oracle.make_reject_given(y, [tuple(s) for s in gold["dpo"]["spans"]])
    Pq = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    lo, acc_o, l1o, l2o = gpt_oracle.forward_dpo(Pq, x, xl, y, yl, bert, ry, ryl, m)
    lo.backward()
    loss, acc = net.forward(x.to(DEV), xl.to(DEV), y.to(DEV), yl.to(DEV), bert.to(DEV), reject=(ry.to(DEV), ryl.to(DEV)))
    named = list(net.named_parameters())
    grads = torch.autograd.grad(loss, [p for _, p in named])
    out.append(("dpo loss vs oracle", abs(float(loss.detach()) - float(lo)) / abs(float(lo)), TOL_NET))
    out.append(("dpo loss vs reference golden", abs(float(loss.detach()) - gold["dpo"]["loss"]) / abs(gold["dpo"]["loss"]), TOL_NET))
    out.append(("dpo loss_2 term vs oracle", abs(float(net.last_dpo[1]) - float(l2o)) / (abs(float(l2o)) + 1e-6), 5e-2))
    out.append(("dpo acc vs reference golden", abs(float(acc) - gold["dpo"]["acc"]), 2.0 / (gold["B"] * gold["Y"])))
    num = den = 0.0
    for (n, _), gk in zip(named, grads):
        if n.endswith(".alpha"):
            continue
        num += float((gk.cpu().double() - Pq[n].grad.double()).pow(2).sum()); den += float(Pq[n].grad.double().pow(2).sum())
    out.append(("dpo grads global", math.sqrt(num / den), KINK_TOL))
    g = _gen(3)
    r2, r2l = make_reject_y(y, yl, generator=g)
    ok = all(int(r2l[b]) >= y.shape[1] and int(r2l[b]) <= 2 * y.shape[1] for b in range(len(yl))) and r2.shape[1] == int(r2l.max())
    out.append(("make_reject_y: repeat-span shape contract", 0.0 if ok else 1.0, 0.0))
    # ---- trainer end to end
    from easevoice_trainer_b200.train.gpt import GPTTrain, GPTTrainParams
    from easevoice_trainer_b200.train import data_gpt
    import yaml
    with tempfile.TemporaryDirectory() as td:
        inp = os.path.join(td, "in"); os.makedirs(os.path.join(inp, "3-bert"))
        table = {f"p{i}": i for i in range(732)}
        rnd = _gen(11)
        with open(os.path.join(inp, "2-name2text.txt"), "w") as f2, open(os.path.join(inp, "6-name2semantic.tsv"), "w") as f6:
            f6.write("item_name\tsemantic_audio\n")
            for i in range(12):
                nph = int(torch.randint(8, 20, (1,), generator=rnd))
                nsem = int(nph * 25 / float(torch.randint(5, 12, (1,), generator=rnd)))
                ph = " ".join(f"p{int(v)}" for v in torch.randint(0, 732, (nph,), generator=rnd))
                f2.write(f"utt{i}\t{ph}\tw2p\tnorm text\n")
                f6.write(f"utt{i}\t" + " ".join(str(int(v)) for v in torch.randint(0, 1024, (nsem,), generator=rnd)) + "\n")
                if i % 2 == 0:
                    torch.save(torch.randn(1024, nph, generator=rnd), os.path.join(inp, "3-bert", f"utt{i}.pt"))
        cfg = yaml.safe_load(open(os.path.join(ROOT, "configs", "gpt.yaml")))
        cfg["model"]["n_layer"] = 2
        cpath = os.path.join(td, "gpt.yaml")
        yaml.safe_dump(cfg, open(cpath, "w"))
        ds = data_gpt.Text2SemanticDataset(os.path.join(inp, "2-name2text.txt"), os.path.join(inp, "6-name2semantic.tsv"),
                                           max_sec=54, phoneme_table=table)
        params = GPTTrainParams(batch_size=24, total_epochs=2, save_every_epoch=1, gpu_ids="0", model_path="", train_input_dir=inp,
                                output_model_name="tiny", project_dir=td)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            res = GPTTrain(params, dataset=ds, config_path=cpath).train()
        lines = [l for l in buf.getvalue().splitlines() if l.startswith("loss-of-easevoice")]
        rec = [json.loads(l[len("loss-of-easevoice"):]) for l in lines]
        out.append(("GPTTrain: one loss line per step with acc/lr/epoch", 0.0 if rec and all(k in rec[0] for k in ("step", "loss", "acc", "lr", "epoch")) else 1.0, 0.0))
        out.append(("GPTTrain: loss finite", 0.0 if all(math.isfinite(r["loss"]) for r in rec) else 1.0, 0.0))
        files = sorted(os.listdir(res.model_path))
        ck = os.listdir(os.path.join(res.model_path, "logs", "ckpt"))
        ok = "tiny-e1.ckpt" in files and "tiny-e2.ckpt" in files and len(ck) == 1 and ck[0].startswith("epoch=1-step=")
        out.append(("GPTTrain: output layout (<name>-e{E}.ckpt + logs/ckpt/epoch=E-step=S.ckpt, latest only)", 0.0 if ok else 1.0, 0.0))
        w = torch.load(os.path.join(res.model_path, "tiny-e2.ckpt"), map_location="cpu", weights_only=False)
        okw = all(k.startswith("model.") and v.dtype == torch.float16 for k, v in w["weight"].items()) and w["info"] == "GPT-e2" and "config" in w
        out.append(("GPTTrain: export = fp16 weights under 'model.' + config + info", 0.0 if okw else 1.0, 0.0))
        # resume: a third epoch continues from epoch=1 (loads weights + ScaledAdam state)
        params.total_epochs = 3
        buf2 = io.StringIO()
        with contextlib.redirect_stdout(buf2):
            GPTTrain(params, dataset=ds, config_path=cpath).train()
        rec2 = [json.loads(l[len("loss-of-easevoice"):]) for l in buf2.getvalue().splitlines() if l.startswith("loss-of-easevoice")]
        out.append(("GPTTrain: resume runs only the missing epoch", 0.0 if rec2 and all(r["epoch"] == 2 for r in rec2) else 1.0, 0.0))
    return out


def check_gemm_tma():
    """TMA-fed persistent wgmma GEMM (csrc/gemm_tma.cu): direct entry point + the Linear dispatch path."""
    from easevoice_trainer_b200 import ops
    out = []
    if PRECISE_MODE[0]:
        return out
    g = _gen(21)
    for tag, M, N, K, splits, epi in (("tails", 1000, 300, 100, 1, False), ("ffn", 4096, 512, 2048, 1, True),
                                       ("wide", 2500, 1536, 512, 1, True), ("narrow N=96", 3000, 96, 256, 1, False),
                                       ("multi-tile persistent", 40000, 512, 96, 1, False),
                                       ("split-K wgrad shape", 512, 384, 8192, 8, False), ("split-K ragged", 200, 130, 1000, 5, False)):
        a = torch.randn(M, K, generator=g)
        b = torch.randn(N, K, generator=g) / math.sqrt(K)
        bias = torch.randn(N, generator=g) if epi else None
        res = torch.randn(M, N, generator=g) if epi else None
        ref = a.double() @ b.double().t()
        if epi:
            ref = torch.relu(ref + bias.double() + res.double())
        init = torch.randn(M, N, generator=g) if splits > 1 else None
        o = ops.gemm_tf32(a.to(DEV), b.to(DEV), out=init.to(DEV) if init is not None else None, bias=bias.to(DEV) if epi else None,
                          res=res.to(DEV) if epi else None, act=ops.ACT_RELU if epi else ops.ACT_NONE, splits=splits)
        if init is not None:
            ref = ref + init.double()
        out.append((f"gemm_tma {tag} M{M} N{N} K{K} s{splits}", rel(o, ref), TOL_TC))
    # Linear through evk_gconv_fwd (eligible shapes dispatch to the TMA kernel), with autograd
    B, T, C, N = 8, 300, 512, 1536
    x = torch.randn(B, T, C, generator=g)
    w = torch.randn(N, C, generator=g) / math.sqrt(C)
    bias = torch.randn(N, generator=g) * 0.1
    gy = torch.randn(B, T, N, generator=g)
    xr, wr, br = [t.clone().requires_grad_(True) for t in (x, w, bias)]
    yr = F.linear(xr, wr, br)
    yr.backward(gy)
    xd, wd, bd = [t.to(DEV).requires_grad_(True) for t in (x, w, bias)]
    y = ops.linear(xd, ops.pack_weight(wd), bd)
    y.backward(gy.to(DEV))
    out.append(("linear via TMA gemm y", rel(y, yr), TOL_TC))
    out.append(("linear via TMA gemm dx", rel(xd.grad, xr.grad), TOL_TC))
    out.append(("linear via TMA gemm dw", rel(wd.grad, wr.grad), TOL_TC))
    out.append(("linear via TMA gemm dbias", rel(bd.grad, br.grad), TOL_F32 * 10))
    return out


def check_vocoder_cfg5():
    """BASELINE.json configs[4] shapes (vocoder only): Generator z [B, 192, 75] -> y_hat [B, 1, 48 000] (1 s at the 48 kHz
    label), MultiPeriodDiscriminator on (y, y_hat), GAN + feature-matching losses and their gradients.  B = 2 here so the
    CPU oracle finishes in seconds; every layer runs at its full 1-s length (the TMA conv / strided-phase / ConvTranspose
    paths at production sizes)."""
    from easevoice_trainer_b200 import ops
    out = []
    net_g, net_d, PG, PD = _load_models()
    B, T = 2, 75
    g = _gen(55)
    z = torch.randn(B, 192, T, generator=g)
    ge = torch.randn(B, 512, 1, generator=g) * 0.5
    y = torch.rand(B, 1, T * 640, generator=g) - 0.5
    zr = z.clone().requires_grad_(True)
    PDr = {k: v.clone().requires_grad_(True) for k, v in PD.items()}
    yh_o = s2_oracle.generator(PG, "dec", zr, ge)
    rs, gs, frs, fgs = s2_oracle.mpd(PDr, y, yh_o)
    loss_o = s2_oracle.generator_loss(gs) + s2_oracle.feature_loss(frs, fgs) + s2_oracle.discriminator_loss(rs, gs)
    loss_o.backward()
    zd = cl(z).requires_grad_(True)
    yh = net_g._generator(zd, cl(ge))                                    # [B, 48000, 1]
    out.append(("cfg5 generator y_hat [B, 48000]", rel(yh.reshape(B, -1), yh_o.reshape(B, -1)), TOL_NET))
    outs = net_d.forward_cl(cl(y), yh)
    lg = lf = ld = 0.0
    for d_i, (logit, fmap) in enumerate(outs):
        # logits of a random-init discriminator on a 0.06-amplitude waveform are small differences of large terms: the
        # relative error of the 6-layer chain is amplified (measured 5e-4 .. 1.1e-2), the loss below pins the absolute scale
        out.append((f"cfg5 D[{d_i}] logits", rel(logit[B:].reshape(B, -1), gs[d_i]), KINK_TOL))
        lg = lg + ops.mean_sq_one_minus(logit[B:])
        ld = ld + ops.mean_sq_one_minus(logit[:B]) + ops.mean_sq(logit[B:])
        for f in fmap:
            lf = lf + ops.mean_abs_diff(f[B:], f[:B])
    loss = lg + 2.0 * lf + ld
    names = [n for n, _ in net_d.named_parameters()]
    grads = torch.autograd.grad(loss, [zd] + [p for _, p in net_d.named_parameters()])
    out.append(("cfg5 loss (gen + fm + disc)", abs(float(loss.detach()) - float(loss_o)) / abs(float(loss_o)), TOL_NET))
    # dz crosses ~60 leaky-ReLU layers at 48 000 positions: kink flips accumulate (measured 4.7e-2; an indexing error in any
    # data-gradient path would give O(1))
    out.append(("cfg5 dz (through D and the whole generator)", rel(cf(grads[0]), zr.grad), NET_GRAD_TENSOR))
    num = den = 0.0
    for n, gk in zip(names, grads[1:]):
        r = PDr[n].grad
        num += float((gk.cpu().double() - r.double()).pow(2).sum()); den += float(r.double().pow(2).sum())
    out.append(("cfg5 D parameter gradients (global)", math.sqrt(num / den), KINK_TOL))
    return out


# ------------------------------------------------------------------------------------------------
# Full-size parity: the benchmarked shapes, through the SAME captured CUDA graph bench.py replays
# ------------------------------------------------------------------------------------------------
REPORT = {}          # tag -> per-tensor error table (run_gpu_checks.py dumps it to gpurun_out/parity_table.json)


def _oracle_threads():
    """torch's intra-op pool stops scaling (and then collapses) on these conv shapes well before the host's core count."""
    n = max(1, min(os.cpu_count() or 1, 16))
    torch.set_num_threads(n)
    return n


def check_s2_full(tag="cfg3"):
    """BASELINE config 3 shapes (T = 346 frames, 120 phonemes, B = 8: every launch takes the same kernel family as the
    benchmarked B = 16).  Losses, forward tensors and EVERY parameter gradient of the graph-replayed step (lr forced to 0 so
    the D update inside the step leaves the weights the oracle sees) vs the CPU oracle, plus the reference's own numbers
    from tests/golden/s2_<tag>.json (written by oracle/pin_against_reference.py --full from the imported reference)."""
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.train import s2_step
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", f"s2_{tag}.json")))
    c = gold["cfg"]
    B, T, X = c["B"], c["T"], c["X"]
    net_g, net_d, PG, PD = _load_models(c["g_seed"], c["d_seed"])                # eval(): dropout off, like the pin
    wav, ssl, text, spec_len, text_len = s2_oracle.synthetic_batch(B, T, X, c["batch_seed"], c["ragged"])
    spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, 640, 2048)
    g = _gen(c["noise_seed"])
    noise = torch.randn(B, 192, T, generator=g)
    ids = (torch.rand(B, generator=g) * (spec_len - 32 + 1)).long()
    assert ids.tolist() == gold["ids_slice"] and spec_len.tolist() == gold["spec_len"]
    # ---- ours first (GPU work overlaps nothing; keeps the CPU oracle's memory high-water mark out of the way)
    stepper = s2_step.S2Step(net_g, net_d, dict(s2_oracle.S2_TRAIN), dict(s2_oracle.S2_DATA))
    stepper.set_lr(0.0)
    batch = dict(ssl=cl(ssl), spec=ops.to_channels_last(spec.to(DEV), pad_to=4), lengths=spec_len.to(DEV).to(torch.int32),
                 wav=wav.reshape(B, -1, 1).to(DEV), text=text.to(DEV), text_lengths=text_len.to(DEV).to(torch.int32))
    noise_d, ids_d = cl(noise), ids.to(DEV)
    ops.dispatch_reset()
    stepper.step(batch, noise=noise_d, ids_slice=ids_d)                             # eager: host-side dispatch accounting
    disp = ops.dispatch_stats()
    res = stepper.graph_step(batch, noise=noise_d, ids_slice=ids_d, keep=True)    # capture (+2 warm-ups) + replay
    res = stepper.graph_step(batch, noise=noise_d, ids_slice=ids_d, keep=True)    # pure replay: what bench.py times
    torch.cuda.synchronize()
    fw = {k: cf(v) for k, v in res["forward"].items() if k in ("z", "z_p", "m_p", "logs_p", "m_q", "logs_q", "y_hat", "y_hat_mel", "y_mel", "y")}
    codes = res["forward"]["codes"].cpu()
    ours = {k: float(res[k]) for k in ("loss_disc", "loss_gen_all", "loss_gen", "loss_fm", "loss_mel", "loss_kl")}
    gd = {n: stepper.opt_d.flat_g[o:o + k].view(p.shape).cpu().clone() for n, p, (o, k) in
          ((n, p, stepper.opt_d.slots[n]) for n, p in net_d.named_parameters())}
    gg = {n: stepper.opt_g.flat_g[o:o + k].view(p.shape).cpu().clone() for n, p, (o, k) in
          ((n, p, stepper.opt_g.slots[n]) for n, p in net_g.named_parameters())}
    tot = sum(disp.values())
    tma = disp["fwd_gemm_tma"] + disp["wgrad_gemm_tma"] + disp["gemm_tf32"]
    out.append((f"s2[{tag}] share of contraction flops NOT on gemm_tma_kernel", 1.0 - tma / tot, 0.20))
    # ---- oracle (CPU, fp32)
    nthr = _oracle_threads()
    OG = {k: (v.clone().requires_grad_(True) if k not in s2_oracle.GEN_BUFFERS else v.clone()) for k, v in PG.items()}
    OD = {k: v.clone().requires_grad_(True) for k, v in PD.items()}
    o = s2_oracle.s2_losses(OG, OD, (ssl, spec, spec_len, wav, text, text_len), noise, ids)
    gd_ref = dict(zip(OD.keys(), torch.autograd.grad(o["loss_disc"], list(OD.values()), retain_graph=True)))
    gn = [k for k in OG if k not in s2_oracle.GEN_BUFFERS]
    gg_ref = dict(zip(gn, torch.autograd.grad(o["loss_gen_all"], [OG[k] for k in gn], allow_unused=True)))
    table = dict(cfg=c, oracle_threads=nthr, dispatch_flops=disp, forward={}, losses={}, grad_d={}, grad_g={})
    for k in ("loss_disc", "loss_gen_all", "loss_gen", "loss_fm", "loss_mel", "loss_kl"):
        e_o, e_g = abs(float(o[k]) - gold[k]) / abs(gold[k]), abs(ours[k] - gold[k]) / abs(gold[k])
        out.append((f"s2[{tag}] oracle {k} vs reference golden", e_o, 1e-4))
        out.append((f"s2[{tag}] {k} vs reference golden", e_g, TOL_NET))
        out.append((f"s2[{tag}] {k} vs oracle", abs(ours[k] - float(o[k])) / abs(float(o[k])), TOL_NET))
        table["losses"][k] = dict(ours=ours[k], oracle=float(o[k]), reference=gold[k])
    out.append((f"s2[{tag}] VQ codes mismatches", float((codes != o["codes"]).sum()), 0.5))
    out.append((f"s2[{tag}] VQ codes checksum == reference golden", abs(int(codes.sum()) - gold["codes_sum"]), 0))
    for k in ("z", "z_p", "m_p", "logs_p", "m_q", "logs_q", "y_hat", "y_hat_mel"):
        e = rel(fw[k], o[k])
        table["forward"][k] = e
        out.append((f"s2[{tag}] {k}", e, TOL_NET))
    out.append((f"s2[{tag}] y_mel", rel(fw["y_mel"], o["y_mel"]), 1e-5))
    out.append((f"s2[{tag}] y slice", rel(fw["y"], o["y"]), 1e-12))
    for k in ("z", "z_p", "m_p", "logs_p", "m_q", "logs_q"):                        # the REFERENCE's values, not the oracle's
        gk = torch.tensor(gold[k + "_b0_c5_t100_108"])
        out.append((f"s2[{tag}] {k}[0,5,100:108] vs reference golden", float((fw[k][0, 5, 100:108] - gk).norm() / (gk.norm() + 1e-12)), 3 * TOL_NET))
        out.append((f"s2[{tag}] |{k}| vs reference golden", abs(float(fw[k].norm()) - gold[k + "_norm"]) / gold[k + "_norm"], TOL_NET))
    gk = torch.tensor(gold["y_hat_b1_0_4000_4008"])
    out.append((f"s2[{tag}] y_hat[1,0,4000:4008] vs reference golden", float((fw["y_hat"][1, 0, 4000:4008] - gk).norm() / (gk.norm() + 1e-12)), 10 * TOL_NET))
    for nm, ours_g, ref_g, gold_n, unused_ok in (("D", gd, gd_ref, gold["grad_norms_d"], ()), ("G", gg, gg_ref, gold["grad_norms_g"], s2_step.FROZEN_G)):
        worst, wname, num, den, worst_gold, wg_name = 0.0, "", 0.0, 0.0, 0.0, ""
        for n, gr in ours_g.items():
            if n in unused_ok:
                assert ref_g[n] is None
                continue
            if n.endswith(("conv_k.bias", "w_ks.bias")):       # analytically zero gradients (see pin_against_reference.py)
                continue
            e = rel(gr, ref_g[n])
            table["grad_" + nm.lower()][n] = dict(rel_l2=e, norm=float(gr.norm()), norm_reference=gold_n[n])
            num += float((gr.double() - ref_g[n].double()).pow(2).sum())
            den += float(ref_g[n].double().pow(2).sum())
            if e > worst:
                worst, wname = e, n
            eg = abs(float(gr.norm()) - gold_n[n]) / (gold_n[n] + 1e-30)
            if eg > worst_gold:
                worst_gold, wg_name = eg, n
        out.append((f"s2[{tag}] {nm} param grads worst rel-L2 ({wname})", worst, NET_GRAD_TENSOR))
        out.append((f"s2[{tag}] {nm} param grads global rel-L2", math.sqrt(num / den), NET_GRAD_GLOBAL))
        out.append((f"s2[{tag}] {nm} |grad| of every tensor vs reference golden, worst ({wg_name})", worst_gold, NET_GRAD_TENSOR))
    REPORT[f"s2_{tag}"] = table
    return out


def check_gpt_full(tag="cfg2"):
    """BASELINE config 2 at the benchmarked model size (24 layers, X = 256, Y = 1024, ragged lengths 512..1024, B = 4):
    loss / targets / logits / every parameter gradient of the GRAPH-REPLAYED micro-batch vs the CPU oracle and the
    reference's numbers (tests/golden/gpt_cfg2.json)."""
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    from easevoice_trainer_b200.train.gpt_step import GptStep
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", f"gpt_{tag}.json")))
    m = gold["model"]
    spec = gpt_oracle.gpt_param_spec(m)
    P = gpt_oracle.init_params(spec, gold["param_seed"])
    P["ar_text_position.alpha"].fill_(gold["alpha_text"]); P["ar_audio_position.alpha"].fill_(gold["alpha_audio"])
    net = Text2SemanticDecoder({"model": m}, layer_dropout=0.0)
    net.load_state_dict(P)
    net = net.to(DEV).eval()
    x, xl, y, yl, bert = gpt_oracle.synthetic_gpt_batch(gold["B"], gold["X"], gold["Y"], gold["batch_seed"], gold["ragged"])
    step = GptStep(net)
    step.batch_idx = 1                                   # a micro-batch without optimizer update: flat_g = its gradients
    batch = dict(phoneme_ids=x.to(DEV), phoneme_ids_len=xl.to(DEV), semantic_ids=y.to(DEV), semantic_ids_len=yl.to(DEV),
                 bert_feature=bert.to(DEV))
    ops.dispatch_reset()
    loss, acc = step.graph_step(batch)                   # capture (its warm-ups leave flat_g untouched) + replay
    disp = ops.dispatch_stats()
    torch.cuda.synchronize()
    loss, acc = float(loss), float(acc)
    logits = net.last_logits[..., :m["vocab_size"]].detach().cpu()
    names = [n for n, _ in net.named_parameters()]
    grads = {n: step.opt.flat_g[o:o + k].view(p.shape).cpu().clone() for n, p, (o, k) in
             ((n, p, step.opt.slots[n]) for n, p in net.named_parameters())}
    y_in, tg = net.make_targets(y.to(DEV), yl.to(DEV))
    tot = sum(disp.values())
    out.append((f"gpt[{tag}] share of contraction flops NOT on gemm_tma_kernel", 1.0 - (disp["fwd_gemm_tma"] + disp["wgrad_gemm_tma"] + disp["gemm_tf32"]) / tot, 0.05))
    nthr = _oracle_threads()
    Pq = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    taps = {}
    loss_o, acc_o, logits_o, tg_o = gpt_oracle.forward_old(Pq, x, xl, y, yl, bert, m, taps)
    loss_o.backward()
    out.append((f"gpt[{tag}] targets (pad_y_eos) exact", float((tg.cpu() != tg_o).sum()), 0.0))
    out.append((f"gpt[{tag}] targets checksum == reference golden", abs(int(tg.sum()) - gold["targets_sum"]), 0))
    out.append((f"gpt[{tag}] logits", rel(logits.reshape(logits_o.shape), logits_o), TOL_NET))
    out.append((f"gpt[{tag}] loss vs oracle", abs(loss - float(loss_o)) / abs(float(loss_o)), TOL_NET))
    out.append((f"gpt[{tag}] loss vs reference golden", abs(loss - gold["loss"]) / abs(gold["loss"]), TOL_NET))
    out.append((f"gpt[{tag}] top-3 acc vs reference golden", abs(acc - gold["acc"]), 8.0 / float(yl.sum())))
    table = dict(B=gold["B"], X=gold["X"], Y=gold["Y"], oracle_threads=nthr, dispatch_flops=disp, loss=dict(ours=loss, oracle=float(loss_o), reference=gold["loss"]), grad={})
    worst, wname, num, den, gl, gl_name = 0.0, "", 0.0, 0.0, 0.0, ""
    alpha_rows = []
    for n in names:
        gk, gr = grads[n], Pq[n].grad
        if n.endswith(".alpha"):
            alpha_rows.append((n, abs(float(gk) - float(gr))))
            continue
        r = rel(gk, gr)
        table["grad"][n] = dict(rel_l2=r, norm=float(gk.norm()), norm_reference=gold["grad_norms"][n])
        if r > worst:
            worst, wname = r, n
        num += float((gk.double() - gr.double()).pow(2).sum()); den += float(gr.double().pow(2).sum())
        e = abs(float(gk.norm()) - gold["grad_norms"][n]) / (gold["grad_norms"][n] + 1e-12)
        if e > gl:
            gl, gl_name = e, n
    alpha_tol = 4.0 * max(math.sqrt(num / den), 1e-4) * float(taps["h0"].grad.norm()) * math.sqrt(0.5)
    # d alpha = <dh0, pe>: a zero-mean error of dh0 averages out in the projection (the noise bound), a SCALE error of the
    # gradient stream (LayerNorm's 1/sigma follows the forward scale) does not -- so the gate is the larger of the 4-sigma
    # noise bound and the per-tensor relative gate applied to |d alpha| itself
    for n, e in alpha_rows:
        out.append((f"gpt[{tag}] d{n} (abs; max(noise bound, {NET_GRAD_TENSOR:g} x |d alpha| = {abs(float(Pq[n].grad)):.3g}))", e,
                    max(alpha_tol, NET_GRAD_TENSOR * abs(float(Pq[n].grad)))))
    out.append((f"gpt[{tag}] grads worst tensor ({wname})", worst, 2 * KINK_TOL))
    out.append((f"gpt[{tag}] grads global", math.sqrt(num / den), KINK_TOL))
    out.append((f"gpt[{tag}] |grad| of every tensor vs reference golden, worst ({gl_name})", gl, 2 * KINK_TOL))
    REPORT[f"gpt_{tag}"] = table
    return out


# ------------------------------------------------------------------------------------------------
# the trainer, end to end, on files (SURVEY 8b: class API, files in / out, stdout protocol, TB scalars, resume)
# ------------------------------------------------------------------------------------------------
def make_s2_dataset_dir(root, n_utt=8, seed=0, min_s=1.0, max_s=3.2):
    """Synthetic <train_input_dir> in the layout Normalize writes (normalize.py:65-211): 2-name2text.txt,
    4-cnhubert/<name>.pt f32 [1,768,T50Hz], 5-wav32k/<name> int16 mono 32 kHz."""
    import wave
    import numpy as np
    g = _gen(seed)
    os.makedirs(os.path.join(root, "4-cnhubert"), exist_ok=True)
    os.makedirs(os.path.join(root, "5-wav32k"), exist_ok=True)
    table = {f"p{i}": i for i in range(732)}
    lines = []
    for u in range(n_utt):
        name = f"utt{u:02d}.wav"
        n = int((min_s + (max_s - min_s) * float(torch.rand(1, generator=g))) * 32000)
        pcm = ((torch.rand(n, generator=g) - 0.5) * 20000).to(torch.int16).numpy()
        with wave.open(os.path.join(root, "5-wav32k", name), "wb") as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(32000); w.writeframes(pcm.astype(np.int16).tobytes())
        T = n // 640
        torch.save(torch.randn(1, 768, T, generator=g), os.path.join(root, "4-cnhubert", name + ".pt"))
        nph = 6 + int(torch.randint(0, 30, (1,), generator=g))
        phones = " ".join(f"p{int(i)}" for i in torch.randint(0, 732, (nph,), generator=g))
        lines.append(f"{name}\t{phones}\t1\ttext")
    with open(os.path.join(root, "2-name2text.txt"), "w", encoding="utf8") as f:
        f.write("\n".join(lines) + "\n")
    return table


def check_sovits_train_e2e(gpu_ids="0"):
    """SovitsTrain(params, dataset).train() on files: loss lines every 10 steps, G_/D_latest.pth, export without enc_q,
    TensorBoard scalars of sovits.py:539-568, frozen ssl_proj bit-identical, resume continues from the stored epoch."""
    import contextlib
    import io
    import tempfile
    from easevoice_trainer_b200.train import data as s2data
    from easevoice_trainer_b200.train import s2_step
    from easevoice_trainer_b200.train.sovits import SovitsTrain, SovitsTrainParams
    from easevoice_trainer_b200 import models, configs
    out = []
    tmp = tempfile.mkdtemp(prefix="evk_e2e_")
    old_base = os.environ.get("EASEVOICE_BASE_PATH")
    os.environ["EASEVOICE_BASE_PATH"] = tmp
    try:
        table = make_s2_dataset_dir(os.path.join(tmp, "in"))
        ds = s2data.TextAudioSpeakerLoader(os.path.join(tmp, "in"), phoneme_table=table)
        nb = len(ds) // 4                                                    # 100 replicated items / batch 4 -> 25 steps / epoch
        params = SovitsTrainParams(batch_size=4, total_epochs=2, save_every_epoch=1, gpu_ids=gpu_ids, train_input_dir=os.path.join(tmp, "in"),
                                   output_model_name="e2e", project_dir=tmp)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            res = SovitsTrain(params, dataset=ds).train()
        lines = [json.loads(l.split(" ", 1)[1]) for l in buf.getvalue().splitlines() if l.startswith("loss-of-easevoice")]
        world = len(gpu_ids.split(","))
        steps = 2 * (nb // world)
        if world == 1:                  # spawned ranks write to their own stdout: the line protocol is checked single-process
            out.append(("e2e loss lines every 10 steps", abs(len(lines) - len(range(0, steps, 10))), 0))
            out.append(("e2e loss line keys", 0.0 if all({"step", "loss", "loss/g/total", "loss/d/total", "learning_rate"} <= set(l) for l in lines) else 1.0, 0.0))
            fin = all(math.isfinite(float(l["loss"])) for l in lines)
            out.append(("e2e losses finite", 0.0 if fin else 1.0, 0.0))
        logs = os.path.join(res.model_path, "logs")
        for f in ("G_latest.pth", "D_latest.pth"):
            out.append((f"e2e {f} written", 0.0 if os.path.isfile(os.path.join(logs, f)) else 1.0, 0.0))
        exp = os.path.join(res.model_path, f"e2e_e2_s{steps}.pth")
        out.append(("e2e export written", 0.0 if os.path.isfile(exp) else 1.0, 0.0))
        ex = torch.load(exp, map_location="cpu")
        out.append(("e2e export: fp16, no enc_q, config + info", 0.0 if (all(v.dtype == torch.float16 for v in ex["weight"].values()) and
                    not any("enc_q" in k for k in ex["weight"]) and ex["info"] == f"2epoch_{steps}iteration" and "model" in ex["config"]) else 1.0, 0.0))
        ck = torch.load(os.path.join(logs, "G_latest.pth"), map_location="cpu")
        out.append(("e2e checkpoint iteration == epoch", abs(ck["iteration"] - 2), 0))
        hps = configs.load_s2_config()
        torch.manual_seed(hps["train"]["seed"])
        fresh = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1, hps["train"]["segment_size"] // hps["data"]["hop_length"],
                                      n_speakers=hps["data"]["n_speakers"], **hps["model"]).state_dict()
        for n in s2_step.FROZEN_G:
            out.append((f"e2e frozen {n} bit-identical after {steps} steps", float((ck["model"][n] != fresh[n]).sum()), 0.0))
        moved = float((ck["model"]["dec.conv_pre.weight"] - fresh["dec.conv_pre.weight"]).abs().max())
        out.append(("e2e trained weights moved", 0.0 if moved > 0 else 1.0, 0.0))
        out.append(("e2e optimizer state torch-style (lr in every group)", 0.0 if all("lr" in g and "initial_lr" in g for g in ck["optimizer"]["param_groups"]) else 1.0, 0.0))
        # TensorBoard scalars (sovits.py:539-568: every 5 steps)
        from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
        ea = EventAccumulator(os.path.join(tmp, "tb_logs", "e2e"))
        ea.Reload()
        tags = set(ea.Tags()["scalars"])
        want = {"loss/g/total", "loss/d/total", "learning_rate", "grad_norm_d", "grad_norm_g", "loss/g/fm", "loss/g/mel", "loss/g/kl_ssl", "loss/g/kl"}
        out.append(("e2e TensorBoard scalar tags", float(len(want - tags)), 0.0))
        n_tb = len(ea.Scalars("loss/g/total")) if "loss/g/total" in tags else 0
        out.append(("e2e TensorBoard points every 5 steps", abs(n_tb - len(range(0, steps, 5))), 0))
        # resume: the stored epoch is re-entered (sovits.py:327-343,378), global_step continues from (epoch-1)*len(loader)
        params3 = SovitsTrainParams(batch_size=4, total_epochs=3, save_every_epoch=1, gpu_ids=gpu_ids, train_input_dir=os.path.join(tmp, "in"),
                                    output_model_name="e2e", project_dir=tmp)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            SovitsTrain(params3, dataset=ds).train()
        lines2 = [json.loads(l.split(" ", 1)[1]) for l in buf.getvalue().splitlines() if l.startswith("loss-of-easevoice")]
        if world == 1:
            first = min(int(l["step"]) for l in lines2)
            out.append(("e2e resume continues at the stored epoch's first step", abs(first - ((nb // world + 9) // 10 * 10)), 0))
        ck3 = torch.load(os.path.join(logs, "G_latest.pth"), map_location="cpu")
        out.append(("e2e resumed run saved epoch 3", abs(ck3["iteration"] - 3), 0))
        out.append(("e2e resumed optimizer step count", abs(float(ck3["optimizer"]["state"][0]["step"]) - 4 * (nb // world)), 0))
    finally:
        if old_base is None:
            os.environ.pop("EASEVOICE_BASE_PATH", None)
        else:
            os.environ["EASEVOICE_BASE_PATH"] = old_base
    return out


def check_side_streams():
    """The forward puts the prior encoder, the flow and four of the six discriminators on side streams (models.SIDE_STREAMS).
    Same networks, same batch, streams on vs off: losses and every parameter gradient must agree to atomics noise."""
    from easevoice_trainer_b200 import ops, models
    from easevoice_trainer_b200.train import s2_step
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "s2_ragged.json")))
    c = gold["cfg"]
    B, T, X = c["B"], c["T"], c["X"]
    net_g, net_d, _, _ = _load_models(c["g_seed"], c["d_seed"])
    wav, ssl, text, spec_len, text_len = s2_oracle.synthetic_batch(B, T, X, c["batch_seed"], c["ragged"])
    spec = mel_oracle.spectrogram(wav.squeeze(1), 2048, 640, 2048)
    g = _gen(c["noise_seed"])
    noise = torch.randn(B, 192, T, generator=g)
    ids = (torch.rand(B, generator=g) * (spec_len - 32 + 1)).long()
    stepper = s2_step.S2Step(net_g, net_d, dict(s2_oracle.S2_TRAIN), dict(s2_oracle.S2_DATA))
    batch = dict(ssl=cl(ssl), spec=ops.to_channels_last(spec.to(DEV), pad_to=4), lengths=spec_len.to(DEV).to(torch.int32),
                 wav=wav.reshape(B, -1, 1).to(DEV), text=text.to(DEV), text_lengths=text_len.to(DEV).to(torch.int32))
    res = {}
    old = models.SIDE_STREAMS
    try:
        for on in (True, False, True):
            models.SIDE_STREAMS = on
            r = stepper.losses(batch, noise=cl(noise), ids_slice=ids.to(DEV))
            ld = stepper.d_loss(r)
            lg, _ = stepper.g_loss(r)
            gd = torch.autograd.grad(ld, [p for _, p in net_d.named_parameters()], retain_graph=True, allow_unused=True)
            gg = torch.autograd.grad(lg, [p for _, p in net_g.named_parameters()], allow_unused=True)
            torch.cuda.synchronize()
            res.setdefault(on, []).append((float(ld), float(lg), [t.detach().clone() for t in gd], [None if t is None else t.detach().clone() for t in gg]))
    finally:
        models.SIDE_STREAMS = old
    a, b, a2 = res[True][0], res[False][0], res[True][1]

    def worst(x, y):
        w = 0.0
        for u, v in zip(x, y):
            if u is not None:
                w = max(w, rel(u, v))
        return w
    out.append(("side streams on vs off: loss_disc", abs(a[0] - b[0]) / abs(b[0]), 1e-5))
    out.append(("side streams on vs off: loss_gen_all", abs(a[1] - b[1]) / abs(b[1]), 1e-5))
    out.append(("side streams on vs off: D param grads worst rel-L2", worst(a[2], b[2]), 1e-4))
    out.append(("side streams on vs off: G param grads worst rel-L2", worst(a[3], b[3]), 1e-4))
    out.append(("side streams on, run twice: G param grads worst rel-L2 (atomics noise floor)", worst(a[3], a2[3]), 1e-4))
    return out


def check_normalize_token():
    """SURVEY 8 row f3 (token half): SynthesizerTrn.extract_latent + the 6-name2semantic.tsv writer on the GPU vs the golden
    the REFERENCE produced (tests/golden/extract_latent.json, oracle/pin_against_reference.py --extract-latent).  Bit-exact."""
    import tempfile
    from easevoice_trainer_b200 import normalize_token as nt
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "extract_latent.json")))
    net_g, _, PG, _ = _load_models(gold["g_seed"], 4321)
    g = _gen(gold["ssl_seed"])
    feats = []
    for case in gold["cases"]:
        ssl = torch.randn(1, 768, case["T"], generator=g)
        feats.append(ssl)
        codes = net_g.extract_latent(ssl.to(DEV))
        ok = tuple(codes.shape) == (1, 1, case["T"] // 2) and codes.dtype == torch.int64
        out.append((f"extract_latent T={case['T']}: shape / dtype of the reference contract", 0.0 if ok else 1.0, 0.5))
        out.append((f"extract_latent T={case['T']}: token mismatches vs the reference golden",
                    float(sum(int(a != b) for a, b in zip(codes[0, 0].cpu().tolist(), case["codes"]))), 0.5))
    toks = nt.extract_tokens(net_g, feats, max_batch=3)
    out.append(("extract_tokens (zero-padded batches of 3): token mismatches vs the golden",
                float(sum(int(a != b) for t, c in zip(toks, gold["cases"]) for a, b in zip(t, c["codes"])) +
                      sum(abs(len(t) - len(c["codes"])) for t, c in zip(toks, gold["cases"]))), 0.5))
    with tempfile.TemporaryDirectory() as d:
        hub = os.path.join(d, "4-cnhubert")
        os.makedirs(hub)
        names = [f"utt{i}.wav" for i in range(len(feats))]
        for n, f in zip(names, feats):
            torch.save(f, os.path.join(hub, n + ".pt"))
        lst = os.path.join(d, "refinements.list")
        with open(lst, "w", encoding="utf8") as f:
            f.write("".join(f"/some/dir/{n}|zh|text\n" for n in names))
        tsv = os.path.join(d, "6-name2semantic.tsv")
        n_written = nt.write_semantic_tsv(lst, hub, tsv, net_g)
        lines = open(tsv, encoding="utf8").read().split("\n")
        good = n_written == len(names) and lines[0] == "item_name\tsemantic_audio" and lines[-1] == "" and all(
            lines[1 + i] == names[i] + "\t" + " ".join(str(v) for v in gold["cases"][i]["codes"]) for i in range(len(names)))
        out.append(("6-name2semantic.tsv written from 4-cnhubert/*.pt == the reference's lines", 0.0 if good else 1.0, 0.5))
    return out


def check_decode():
    """SURVEY 8 row f4 (vocoder half): SynthesizerTrn.decode -- quantizer.decode, prior encoder, flow in REVERSE, generator --
    vs the waveform the reference produced with the same injected noise (tests/golden/decode.pt,
    oracle/pin_against_reference.py --decode) and vs the oracle."""
    out = []
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "decode.pt"), weights_only=False)
    c = gold["cfg"]
    net_g, _, PG, _ = _load_models(c["g_seed"], 4321)
    g = _gen(c["seed"])
    codes = torch.randint(0, 1024, (1, 1, c["T"]), generator=g)
    text = torch.randint(0, 300, (1, c["X"]), generator=g)
    refers = [torch.rand(1, 1025, tr, generator=g) * 2.0 for tr in c["Tr"]]
    noise = torch.randn(1, 192, 2 * c["T"], generator=g)
    with torch.no_grad():
        ora = s2_oracle.decode(PG, codes, text, refers, noise, c["noise_scale"])
    out.append(("decode: oracle vs reference golden waveform", rel(ora, gold["wave"]), 1e-5))
    o = net_g.decode(codes.to(DEV), text.to(DEV), [r.to(DEV) for r in refers], noise_scale=c["noise_scale"], noise=noise.to(DEV))
    out.append(("decode: output shape [1, 1, 2T * 640]", 0.0 if tuple(o.shape) == (1, 1, 2 * c["T"] * 640) else 1.0, 0.5))
    out.append(("decode: waveform vs reference golden (rel-L2)", rel(o, gold["wave"]), TOL_NET))
    out.append(("decode: waveform vs oracle (rel-L2)", rel(o, ora), TOL_NET))
    o1 = net_g.decode(codes.to(DEV), text.to(DEV), refers[0].to(DEV), noise_scale=c["noise_scale"], noise=noise.to(DEV))
    with torch.no_grad():
        ora1 = s2_oracle.decode(PG, codes, text, refers[:1], noise, c["noise_scale"])
    out.append(("decode: single reference spectrogram (tensor, not list) vs oracle", rel(o1, ora1), TOL_NET))
    o2 = net_g.decode(codes.to(DEV), text.to(DEV), refers[0].to(DEV))          # internal noise: finite, right shape, not the seeded one
    ok = bool(torch.isfinite(o2).all()) and tuple(o2.shape) == tuple(o1.shape) and float((o2 - o1).abs().max()) > 0.0
    out.append(("decode: internal normal draw when no noise is given", 0.0 if ok else 1.0, 0.5))
    # speed != 1: the prior encoder output is resampled to int(2T / speed) + 1 frames (models.py:246-248)
    Fs = int(2 * c["T"] / c["speed"]) + 1
    noise_s = torch.randn(1, 192, Fs, generator=g)
    os_ = net_g.decode(codes.to(DEV), text.to(DEV), [r.to(DEV) for r in refers], noise_scale=c["noise_scale"], speed=c["speed"],
                       noise=noise_s.to(DEV))
    out.append((f"decode speed={c['speed']}: output shape [1, 1, (int(2T / speed) + 1) * 640]",
                0.0 if tuple(os_.shape) == (1, 1, Fs * 640) else 1.0, 0.5))
    out.append((f"decode speed={c['speed']}: waveform vs reference golden (rel-L2)", rel(os_, gold["wave_speed"]), TOL_NET))
    return out


def check_infer_panel():
    """SURVEY 8 row f4 (AR half): Text2SemanticDecoder.infer_panel -- prompt pass on the training kernels + KV-cache decoding
    (evk_attn_decode_dev) -- greedy, vs the token sequence and logits the REFERENCE decoded (tests/golden/infer_panel.json)."""
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    from oracle import gpt_oracle
    out = []
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "infer_panel.json")))
    c = gold["cfg"]
    m = dict(gpt_oracle.GPT_MODEL, n_layer=c["n_layer"])
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), c["param_seed"])
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    net = Text2SemanticDecoder({"model": m})
    net.load_state_dict(P)
    net = net.to(DEV).eval()
    g = _gen(c["seed"])
    x = torch.randint(0, m["phoneme_vocab_size"], (1, c["X"]), generator=g)
    bert = torch.randn(1, 1024, c["X"], generator=g)
    prompts = torch.randint(0, 1024, (1, c["Yp"]), generator=g)
    # ---- the KV-cache attention kernel alone vs torch
    gg = _gen(5)
    cache = torch.randn(2, 700, 3 * 512, generator=gg).to(DEV)
    for n in (1, 2, 37, 70, 128, 129, 700):                    # row n - 1 appended at n_prev = n - 1: keys 0 .. n - 1
        a = ops_mod().attn_decode_dev(cache.clone(), torch.tensor([n - 1], dtype=torch.int32, device=DEV), 16,
                                      cache[:, n - 1:n].clone())
        q = cache[:, n - 1, :512].view(2, 16, 1, 32).double().cpu()
        k = cache[:, :n, 512:1024].reshape(2, n, 16, 32).permute(0, 2, 1, 3).double().cpu()
        v = cache[:, :n, 1024:].reshape(2, n, 16, 32).permute(0, 2, 1, 3).double().cpu()
        ref = (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(32.0), -1) @ v).permute(0, 2, 1, 3).reshape(2, 1, 512)
        out.append((f"attn_decode_dev n_keys={n} vs float64 softmax(q k^T / sqrt(32)) v", rel(a, ref), 2e-6))
    # ---- the skinny Linear of the token step (evk_gemv_rows: exact fp32 over the packed, TF32-rounded weight) vs float64
    o = ops_mod()
    for rows, N, C, act in ((1, 1536, 512, o.ACT_NONE), (1, 512, 2048, o.ACT_NONE), (1, 2048, 512, o.ACT_RELU), (3, 1028, 512, o.ACT_NONE),
                            (4, 96, 64, o.ACT_LRELU), (2, 513, 260, o.ACT_NONE)):
        wv = (torch.randn(N, C, 1, generator=gg) / math.sqrt(C)).to(DEV)
        bv = torch.randn(N, generator=gg).to(DEV)
        xv = torch.randn(1, rows, C, generator=gg).to(DEV)
        pw = o.pack_weight(wv, None, need_pb=False)
        with torch.no_grad():
            yv = o.linear(xv, pw, bv, act=act, slope=0.1)
        wr = pw.pa[0, :N, :C].double().cpu()                     # the operand the kernel reads (rounded to TF32 at pack time)
        ref = xv[0].double().cpu() @ wr.t() + bv.double().cpu()
        ref = torch.relu(ref) if act == o.ACT_RELU else (torch.where(ref > 0, ref, 0.1 * ref) if act == o.ACT_LRELU else ref)
        out.append((f"gemv_rows rows={rows} N={N} C={C} act={act} vs float64 on the packed weight", rel(yv[0], ref), 2e-6))
        out.append((f"gemv_rows rows={rows} N={N} C={C} vs the unrounded weight (TF32 weight rounding only)",
                    rel(yv[0], torch.relu(xv[0].double().cpu() @ wv[:, :, 0].double().cpu().t() + bv.double().cpu()) if act == o.ACT_RELU else
                        (lambda r: torch.where(r > 0, r, 0.1 * r) if act == o.ACT_LRELU else r)(xv[0].double().cpu() @ wv[:, :, 0].double().cpu().t() + bv.double().cpu())), TOL_TC))
    # ---- LayerNorm(x + res) of a handful of rows (block-per-row kernel of the token step) vs float64
    for rows, C in ((1, 512), (3, 768), (8, 1000)):
        xv, rv = torch.randn(1, rows, C, generator=gg) * 2 + 0.3, torch.randn(1, rows, C, generator=gg)
        gm, bt = 1 + 0.1 * torch.randn(C, generator=gg), 0.1 * torch.randn(C, generator=gg)
        with torch.no_grad():
            yv = o.layernorm(xv.to(DEV), gm.to(DEV), bt.to(DEV), res=rv.to(DEV))
        ref = torch.nn.functional.layer_norm((xv + rv).double(), (C,), gm.double(), bt.double(), 1e-5)
        out.append((f"layernorm rows={rows} C={C} (+res) vs float64", rel(yv, ref), 2e-6))
    # ---- greedy decoding
    tr = []
    y, idx = net.infer_panel(x.to(DEV), torch.tensor([c["X"]], device=DEV), prompts.to(DEV), bert.to(DEV), top_k=c["top_k"], top_p=100,
                             early_stop_num=c["early_stop_num"], temperature=c["temperature"],
                             repetition_penalty=c["repetition_penalty"], trace=tr)
    toks = y[0].cpu().tolist()
    ref_toks = gold["tokens"]
    first_bad = next((i for i, (a, b) in enumerate(zip(toks, ref_toks)) if a != b), None)
    if first_bad is None and len(toks) == len(ref_toks):
        out.append(("infer_panel greedy: token sequence == the reference's (prompt + 40 generated)", 0.0, 0.5))
        out.append(("infer_panel: index of the last generated token", abs(int(idx) - gold["idx"]), 0.5))
    else:
        # a TF32 Linear stack may flip an argmax only where the reference's own top-2 margin is inside the rounding noise
        step = (first_bad if first_bad is not None else min(len(toks), len(ref_toks))) - c["Yp"]
        margin = gold["top2_margin"][step] if 0 <= step < len(gold["top2_margin"]) else 1e9
        out.append((f"infer_panel greedy: first divergence at step {step} has a reference top-2 margin {margin:.2e} < 2e-2", margin, 2e-2))
    for s_, refl in gold["logits_step"].items():
        s_i = int(s_)
        if s_i < len(tr) and (first_bad is None or s_i <= first_bad - c["Yp"]):
            out.append((f"infer_panel logits of step {s_i} vs reference (rel-L2)", rel(tr[s_i][0], torch.tensor(refl)), TOL_NET))
    # sampling path (top_k = 5, temperature 0.8): runs, stops at early_stop_num, tokens in range
    y2, idx2 = net.infer_panel(x.to(DEV), torch.tensor([c["X"]], device=DEV), prompts.to(DEV), bert.to(DEV), top_k=5, top_p=0.9,
                               early_stop_num=12, temperature=0.8)
    ok = y2.shape[1] <= c["Yp"] + 13 and int(y2.max()) <= 1024 and torch.equal(y2[:, :c["Yp"]].cpu(), prompts)
    out.append(("infer_panel sampling (top_k 5, top_p 0.9, T 0.8, early stop 12): prompt kept, length bounded, ids in range", 0.0 if ok else 1.0, 0.5))
    return out


def ops_mod():
    from easevoice_trainer_b200 import ops
    return ops


def check_hubert():
    """SURVEY 8 row f3 (ssl half): the HuBERT forward of Normalize.ssl on the library's kernels vs the output transformers'
    HubertModel produced from the same seeded weights (tests/golden/hubert.pt, oracle/pin_against_reference.py --hubert)."""
    from easevoice_trainer_b200 import hubert, ops
    from oracle import hubert_oracle as ho
    out = []
    g = _gen(3)
    x = torch.randn(2, 301, 70, generator=g) * 2.0 + 0.5
    gm, bt = 1.0 + 0.1 * torch.randn(70, generator=g), 0.1 * torch.randn(70, generator=g)
    ref = torch.nn.functional.group_norm(x.transpose(1, 2).double(), 70, gm.double(), bt.double(), 1e-5).transpose(1, 2)
    out.append(("instnorm_cl vs GroupNorm(C, C) (float64)", rel(ops.instnorm_cl(x.to(DEV), gm.to(DEV), bt.to(DEV)), ref), 2e-6))
    out.append(("instnorm_cl + GELU", rel(ops.instnorm_cl(x.to(DEV), gm.to(DEV), bt.to(DEV), gelu_after=True),
                                          torch.nn.functional.gelu(ref)), 2e-6))
    out.append(("gelu (erf) vs float64", rel(ops.gelu(x.to(DEV)), torch.nn.functional.gelu(x.double())), 1e-6))
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "hubert.pt"), weights_only=False)
    for c in gold["cases"]:
        m = dict(ho.HUBERT_BASE, layers=c["layers"])
        P = ho.init_params(ho.param_spec(m), c["param_seed"])
        net = hubert.HubertModel({"num_hidden_layers": c["layers"]})
        net.load_state_dict(P)
        net = net.to(DEV).eval()
        wav = torch.randn(1, c["L"], generator=_gen(c["wav_seed"])) * c["wav_scale"]
        o = net(wav.to(DEV))["last_hidden_state"]
        out.append((f"hubert[{c['tag']}] output shape", 0.0 if tuple(o.shape) == tuple(c["out"].shape) else 1.0, 0.5))
        out.append((f"hubert[{c['tag']}] last_hidden_state vs transformers golden (rel-L2)", rel(o, c["out"]), TOL_NET))
        if c["tag"] == "l2":
            taps = {}
            with torch.no_grad():
                ho.forward(P, wav, m, taps=taps)
            # the feature extractor alone (7 strided convs + GroupNorm + GELU): recomputed through the public pieces
            with net.inference_weights():
                xx = ops.pad_channels(wav.to(DEV).unsqueeze(-1).contiguous(), 4)
                for i, (k, st) in enumerate(zip(net.cfg["conv_kernel"], net.cfg["conv_stride"])):
                    xx = ops.conv(xx, net.w(f"feature_extractor.conv_layers.{i}.conv", need_pb=False, pad1=4 if i == 0 else 0), None, stride=st)
                    xx = ops.instnorm_cl(xx, net.P("feature_extractor.conv_layers.0.layer_norm.weight"),
                                         net.P("feature_extractor.conv_layers.0.layer_norm.bias"), 1e-5, gelu_after=True) if i == 0 else ops.gelu(xx)
            out.append(("hubert[l2] feature extractor output vs oracle (rel-L2)", rel(xx, taps["features"]), TOL_NET))
    return out


ALL = [check_conv, check_conv_transpose, check_elementwise, check_attention, check_vq_losses_optim, check_mel,
       lambda: check_s2("small"), lambda: check_s2("ragged"), check_api_layouts,
       check_gpt_kernels, check_scaled_adam, lambda: check_gpt("small"), lambda: check_gpt("ragged"),
       check_gpt_dpo_and_trainer, check_gemm_tma, check_vocoder_cfg5,
       lambda: check_s2_full("cfg3"), lambda: check_s2_full("cfg3r"), lambda: check_gpt_full("cfg2"),
       check_sovits_train_e2e, check_stft, check_fused_dropout, check_side_streams, check_normalize_token, check_decode, check_infer_panel, check_hubert]
NAMES = ["conv", "conv_transpose", "elementwise", "attention", "vq_losses_optim", "mel", "s2_small", "s2_ragged", "api",
         "gpt_kernels", "scaled_adam", "gpt_small", "gpt_ragged", "gpt_dpo_trainer", "gemm_tma", "vocoder_cfg5",
         "s2_cfg3", "s2_cfg3r", "gpt_cfg2", "sovits_train_e2e", "stft_mrstft", "fused_dropout", "side_streams", "normalize_token", "decode", "infer_panel", "hubert"]
