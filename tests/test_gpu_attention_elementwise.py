"""Every output of the mma.sync attention kernels (csrc/attn_mma.cuh under flash.cu and attn64.cu) against float64, element
for element, in TF32 and in 3xTF32 mode.

The operands are small integers (tests/attention_ref.py states the error model), so each output has a first-order error
bound from the kernels' rounding rules alone; the gate is SAFETY times that bound.  Masked and dropped probabilities are
exact (ex2(-inf) = 0, 0.f) and must be 0.0.  A probe V that is the identity on one key block per head makes one launch
return the probability of every (query, key) pair, so a key wrongly admitted or dropped at a tile, prefix, x_len, y_len or
lens boundary shows as one wrong element -- which a whole-tensor relative-L2 gate averages away.
"""
import ctypes
import math

import pytest
import torch

from tests import attention_ref as A

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
SCALE_FLASH, SCALE_64 = 1.0 / math.sqrt(A.FLASH_DK), 0.125
WORST = {}


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    L = lib.init()
    L.evk_set_precise(0)
    try:
        yield ops
    finally:
        L.evk_set_precise(0)
        for k in sorted(WORST):
            print(f"worst err / gate  {k}: {WORST[k]:.3f}")


@pytest.fixture(params=list(A.MODES))
def mode(request, ops):
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1 if request.param == "3xtf32" else 0)
    try:
        yield request.param
    finally:
        lib.init().evk_set_precise(0)


def check(got, ref, model, what, axes, tiles, zero=None, keys=None, key_tile=None):
    """|got - ref| <= SAFETY * model and finite at every element, and got == 0.0 exactly where `zero` is set.  The report
    lists the first mismatches as coordinates with the tile each falls in; for a readout (axes b, i, h, c) `keys` maps
    (h, c) to the key j it reads, reported with its key tile."""
    got = got.detach().double().cpu()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    r = A.ratio(got, ref, model)
    bad = A.outside_gate(got, ref, model, zero)
    n = int(bad.sum())
    if n:
        lines = []
        for idx in bad.nonzero()[:8].tolist():
            coord = ", ".join(f"{a}={i}" + (f" (tile {i // tiles[a]})" if a in tiles else "") for a, i in zip(axes, idx))
            if keys is not None:
                j = int(keys[idx[axes.index("h")], idx[axes.index("c")]])
                coord += f", key j={j} (key tile {j // key_tile})" if j >= 0 else ", key past L"
            lines.append(f"  [{coord}] got {float(got[tuple(idx)])!r} want {float(ref[tuple(idx)])!r} "
                         f"gate {A.SAFETY * float(model[tuple(idx)]):.3g}")
        pytest.fail(f"{what}: {n} of {bad.numel()} outputs outside the gate\n" + "\n".join(lines))
    kernel = what.split(" ")[0]
    w = float(r.max()) if r.numel() else 0.0
    WORST[kernel] = max(WORST.get(kernel, 0.0), w)
    return w


# ---- flash ABI --------------------------------------------------------------------------------------------------------
def pack(q, k, v):
    """[B, H, L, d] x 3 -> qkv [B, L, 3 H d] as the GPT's in_proj lays it out"""
    B, H, L, d = q.shape
    return torch.cat([t.transpose(1, 2).reshape(B, L, H * d) for t in (q, k, v)], -1).float().contiguous()


def flash_fwd(ops, qkv, H, X, xl, yl, p=0.0, sid=A.DROP_SID):
    B, L, D3 = qkv.shape
    D = D3 // 3
    qkv = qkv.to(DEV)
    out = torch.empty(B, L, D, device=DEV)
    lse = torch.empty(B * H, L, device=DEV)
    base = qkv.data_ptr()
    xl, yl = xl.to(DEV), yl.to(DEV)
    ops._call("evk_flash_attn_fwd", base, base + 4 * D, base + 8 * D, D3, ops._p(out), D, ops._p(lse), B, H, L, X, A.FLASH_DK,
              ops._p(xl), ops._p(yl), ctypes.c_float(1.0 / math.sqrt(A.FLASH_DK)), ctypes.c_float(p),
              ops._p(ops.rng_state(DEV)), ctypes.c_uint64(sid))
    return qkv, out, lse.view(B, H, L)


def flash_bwd(ops, qkv, out, lse, dout, H, X, xl, yl, p=0.0, sid=A.DROP_SID, pad_o=0):
    """evk_flash_attn_bwd; pad_o > 0 passes O with row pitch D + pad_o (pitch % 4 == 2: the one-warp-per-row delta kernel)"""
    B, L, D3 = qkv.shape
    D = D3 // 3
    o = out
    if pad_o:
        o = torch.full((B, L, D + pad_o), float("nan"), device=DEV)
        o[..., :D] = out
    dout = dout.float().to(DEV).contiguous()
    dqkv = torch.full_like(qkv, float("nan"))
    delta = torch.empty(B * H, L, device=DEV)
    base, dbase = qkv.data_ptr(), dqkv.data_ptr()
    xl, yl = xl.to(DEV), yl.to(DEV)
    ops._call("evk_flash_attn_bwd", base, base + 4 * D, base + 8 * D, D3, ops._p(o), D + pad_o, ops._p(lse), ops._p(dout), D,
              ops._p(delta), dbase, dbase + 4 * D, dbase + 8 * D, D3, B, H, L, X, A.FLASH_DK, ops._p(xl),
              ops._p(yl), ctypes.c_float(1.0 / math.sqrt(A.FLASH_DK)), ctypes.c_float(p), ops._p(ops.rng_state(DEV)),
              ctypes.c_uint64(sid))
    return [t.view(B, L, H, A.FLASH_DK).transpose(1, 2).cpu() for t in dqkv.split(D, -1)]


FLASH_AXES, FLASH_TILES = ("b", "i", "h", "c"), {"i": A.FLASH_TILE}


def _flash_readout(ops, mode, X, Y, xl, yl, seed):
    L = X + Y
    B = len(xl)
    H = -(-L // A.FLASH_DK)
    q, k = A.readout_qk(B, L, A.FLASH_DK, seed)
    vis = A.flash_visible(xl, yl, X, L)
    ref, model, P = A.readout_ref(q[:, None], k[:, None], vis, SCALE_FLASH, mode, A.FLASH_TILE)
    keys = A.readout_keys(L, H, A.FLASH_DK)
    V = A.readout_v(L, H, A.FLASH_DK)
    qkv = torch.cat([q.repeat(1, 1, H), k.repeat(1, 1, H), V[None].expand(B, L, H * A.FLASH_DK)], -1).float().contiguous()
    _, out, _ = flash_fwd(ops, qkv, H, X, xl, yl)
    got = out.cpu().view(B, L, H, A.FLASH_DK)
    zero = A.gather_readout(vis.double(), keys) == 0
    return check(got, A.gather_readout(ref[:, 0], keys), A.gather_readout(model[:, 0], keys), f"flash_fwd readout {mode} X={X} Y={Y}",
                 FLASH_AXES, FLASH_TILES, zero, keys, A.FLASH_TILE)


# ---- a. probability readout of the mask ---------------------------------------------------------------------------------
@pytest.mark.parametrize("X", A.FLASH_READOUT_X)
def test_flash_mask_readout(ops, mode, X):
    worst = 0.0
    for Y in A.FLASH_READOUT_Y:
        xl, yl = A.flash_lens(X, Y)
        worst = max(worst, _flash_readout(ops, mode, X, Y, xl, yl, 100 * X + Y))
    print(f"flash readout X={X} {mode}: worst err / gate {worst:.3f}")


def test_flash_mask_readout_shipped_shape(ops, mode):
    X, Y, xl, yl = A.FLASH_SHIPPED
    w = _flash_readout(ops, mode, X, Y, torch.tensor(xl), torch.tensor(yl), 7)
    print(f"flash readout shipped {mode}: worst err / gate {w:.3f}")


@pytest.mark.parametrize("L", A.PAD_READOUT_L)
def test_attn_pad_mask_readout(ops, mode, L):
    lens = torch.tensor([min(n, L) for n in A.PAD_LENS + (L,)])
    B = len(lens)
    H = -(-L // A.ATTN64_DK)
    q, k = A.readout_qk(B, L, A.ATTN64_DK, L)
    vis = A.pad_visible(lens, L)
    ref, model, _ = A.readout_ref(q[:, None], k[:, None], vis, SCALE_64, mode, A.ATTN64_KEY_TILE)
    keys = A.readout_keys(L, H, A.ATTN64_DK)
    V = A.readout_v(L, H, A.ATTN64_DK)
    qkv = torch.cat([q.repeat(1, 1, H), k.repeat(1, 1, H), V[None].expand(B, L, H * A.ATTN64_DK)], -1).float().to(DEV)
    out = ops.attention_pad(qkv, heads=H, lens=lens.to(DEV), scale=SCALE_64).cpu().view(B, L, H, A.ATTN64_DK)
    zero = A.gather_readout(vis.double(), keys) == 0
    w = check(out, A.gather_readout(ref[:, 0], keys), A.gather_readout(model[:, 0], keys), f"attn64_pad readout {mode} L={L}",
              ("b", "i", "h", "c"), {"i": 64}, zero, keys, A.ATTN64_KEY_TILE)
    print(f"attn64 pad readout L={L} {mode}: worst err / gate {w:.3f}")


# ---- b. dropout ---------------------------------------------------------------------------------------------------------
def _seed_rng(ops):
    """RNG state (DROP_SEED, 0): the state tests/test_cpu_attention_ref.py rehearses the keep masks with"""
    ops.manual_seed(A.DROP_SEED, DEV)
    state = ops.rng_state(DEV).clone()
    assert state.cpu().tolist() == [A.DROP_SEED, 0]
    return state


@pytest.mark.parametrize("p", A.DROP_P)
def test_flash_dropout_readout(ops, mode, p):
    B, X, Y = A.DROP_SHAPE
    L = X + Y
    H = -(-L // A.FLASH_DK)
    nb = H
    xl, yl = torch.tensor([X, X // 2, 1]), torch.tensor([Y, 1, Y - 1])
    q, k = A.readout_qk(B, L, A.FLASH_DK, 11)
    vis = A.flash_visible(xl, yl, X, L)
    state = _seed_rng(ops)
    keep = A.keep_tensor(B, H, L, A.DROP_SEED, 0, A.DROP_SID, p)
    ds = A.drop_scale(keep, p)
    ref, model, _ = A.readout_ref(q[:, None], k[:, None], vis, SCALE_FLASH, mode, A.FLASH_TILE, ds)
    seen = torch.zeros(H, L, dtype=torch.bool)
    worst = 0.0
    for r in range(nb):                                              # rotate the probe blocks: every (head, key) read
        keys = A.readout_keys(L, H, A.FLASH_DK, r)
        V = A.readout_v(L, H, A.FLASH_DK, r)
        qkv = torch.cat([q.repeat(1, 1, H), k.repeat(1, 1, H), V[None].expand(B, L, H * A.FLASH_DK)], -1).float().contiguous()
        _, out, _ = flash_fwd(ops, qkv, H, X, xl, yl, p)
        got = out.cpu().view(B, L, H, A.FLASH_DK)
        kept = A.gather_readout((vis[:, None] & keep).double(), keys) != 0
        zero_got = got == 0
        if not torch.equal(zero_got, ~kept):
            idx = (zero_got != ~kept).nonzero()[:8].tolist()
            pytest.fail(f"flash dropout p={p} {mode} rotation {r}: zero set differs from masked-or-dropped at "
                        f"{[(b, i, h, int(keys[h, c])) for b, i, h, c in idx]}")
        worst = max(worst, check(got, A.gather_readout(ref, keys), A.gather_readout(model, keys),
                                 f"flash_fwd dropout p={p} {mode} rotation {r}", FLASH_AXES, FLASH_TILES, keys=keys,
                                 key_tile=A.FLASH_TILE))
        seen[torch.arange(H)[:, None].expand_as(keys)[keys >= 0], keys[keys >= 0]] = True
    assert bool(seen.all())
    assert torch.equal(ops.rng_state(DEV), state)                  # the launches do not advance the RNG offset
    print(f"flash dropout readout p={p} {mode}: worst err / gate {worst:.3f}")


# ---- c, d. general V: forward and backward ------------------------------------------------------------------------------
@pytest.mark.parametrize("case", A.FLASH_GENERAL, ids=[c[0] for c in A.FLASH_GENERAL])
def test_flash_general_forward_backward(ops, mode, case):
    name, B, H, X, Y, pattern, p = case
    L = X + Y
    q, k, v, do, xl, yl = A.flash_general_inputs(B, H, X, Y, pattern, len(name) * 31 + B)
    vis = A.flash_visible(xl, yl, X, L)[:, None]
    _seed_rng(ops)
    keep = A.keep_tensor(B, H, L, A.DROP_SEED, 0, A.DROP_SID, p) if p else None
    ds = None if keep is None else A.drop_scale(keep, p)
    qr, kr, vr = (t.clone().requires_grad_(True) for t in (q, k, v))
    O, lse, P, t = A.attention_ref(qr, kr, vr, vis, SCALE_FLASH, ds)
    O.backward(do)
    O, lse = O.detach(), lse.detach()
    bO, Else, Et = A.fwd_model(t.detach(), vis, P.detach(), lse, v.abs(), mode, A.FLASH_TILE, dscale=ds)
    qkv, out, lse_k = flash_fwd(ops, pack(q, k, v), H, X, xl, yl, p)
    got_o = out.cpu().view(B, L, H, A.FLASH_DK).transpose(1, 2)
    axes, tiles = ("b", "h", "i", "c"), {"i": A.FLASH_TILE}
    rs = [check(got_o, O, bO, f"flash_fwd O {mode} {name}", axes, tiles),
          check(lse_k.cpu(), lse, Else, f"flash_fwd lse {mode} {name}", ("b", "h", "i"), tiles)]
    bq, bk, bv = A.flash_bwd_model(q, k, v, do, vis, P.detach(), t.detach(), lse, O, bO, Else, Et, SCALE_FLASH, mode, ds)
    dead = torch.zeros(B, 1, L, 1, dtype=torch.bool)                # keys no query may see: exact zero gradients
    for b in range(B):
        dead[b, 0, int(xl[b]):X] = True
        dead[b, 0, X + int(yl[b]):] = True
    for pad_o in ((0, 2) if name == "random" else (0,)):
        dq, dk, dv = flash_bwd(ops, qkv, out, lse_k.reshape(B * H, L), do.transpose(1, 2).reshape(B, L, H * A.FLASH_DK), H, X, xl, yl, p,
                               pad_o=pad_o)
        sfx = f"{mode} {name}" + (" ldo%4==2" if pad_o else "")
        rs += [check(dq, qr.grad, bq, f"flash_dq dQ {sfx}", axes, tiles),
               check(dk, kr.grad, bk, f"flash_dkv dK {sfx}", ("b", "h", "j", "c"), {"j": A.FLASH_TILE},
                     dead.expand_as(dk)),
               check(dv, vr.grad, bv, f"flash_dkv dV {sfx}", ("b", "h", "j", "c"), {"j": A.FLASH_TILE},
                     dead.expand_as(dv))]
    print(f"flash {name} {mode}: worst err / gate O {rs[0]:.3f} lse {rs[1]:.3f} dQ {rs[2]:.3f} dK {rs[3]:.3f} dV {rs[4]:.3f}")


# ---- e. rope attention --------------------------------------------------------------------------------------------------
def _rope_run(ops, q, k, v, gate, cs, layout):
    n, H, L, _ = q.shape
    D = H * 64
    ld = (3 * D + H + 3) // 4 * 4 + 4
    Xs = torch.zeros(n, L, ld, dtype=torch.float64)
    for i, t in enumerate((q, k, v)):
        Xs[..., i * D:(i + 1) * D] = t.permute(0, 2, 1, 3).reshape(n, L, D)
    Xs[..., 3 * D:3 * D + H] = gate.permute(0, 2, 1)
    X = (Xs.permute(1, 0, 2)[None] if layout == "time" else Xs[None]).float().contiguous().to(DEV)   # [1, T, F, ld]
    _, T, Fb, _ = X.shape
    out = torch.full((T * Fb, D + 4), 7.0, device=DEV)
    geo = (1, T * Fb, Fb, 1, Fb) if layout == "time" else (T, Fb, 1, 0, 1)
    ops.rope_attn(X.view(-1, ld), cs.to(DEV).contiguous(), out[:, :D], H, L, *geo)
    assert bool((out[:, D:] == 7).all())
    o = out[:, :D].cpu().view(T, Fb, H, 64)
    o = o.permute(1, 0, 2, 3) if layout == "time" else o                  # [n, L, H, 64]
    return o.permute(0, 2, 1, 3)


@pytest.mark.parametrize("layout", ["time", "freq"])
def test_rope_attn_elementwise(ops, mode, layout):
    from oracle import bs_roformer_oracle as O_
    tables = [(L, A.quarter_turn_cs(L), "quarter") for L in A.ROPE_L]
    tables.append((A.ROPE_REAL_L, torch.stack(O_.rotary_cos_sin(A.ROPE_REAL_L), -1).float(), "rotary"))
    worst = 0.0
    for L, cs, kind in tables:
        q, k, v, gate = A.rope_inputs(2, A.ROPE_H, L, L)
        ref, model = A.rope_ref(q, k, v, gate, cs, mode)
        got = _rope_run(ops, q, k, v, gate, cs, layout)
        worst = max(worst, check(got, ref, model, f"attn64_rope {mode} {layout} {kind} L={L}", ("n", "h", "i", "c"), {"i": 64}))
    print(f"rope {layout} {mode}: worst err / gate {worst:.3f}")
