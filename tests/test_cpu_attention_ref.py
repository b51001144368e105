"""CPU rehearsal of tests/test_gpu_attention_elementwise.py: the float64 references agree with softmax attention as the
existing tests write it, an fp32 emulation of the kernels' arithmetic stays within the first-order error model (half the
gate) at every element of every input the GPU test uses, and the element-wise gate rejects every modelled kernel fault --
some of which the whole-tensor relative-L2 gate (checks.TOL_TC) lets through."""
import math

import pytest
import torch

from tests import attention_ref as A
from tests.checks import TOL_TC, _sdpa_oracle

MODES = tuple(A.MODES)
SCALE_FLASH, SCALE_64 = 1.0 / math.sqrt(A.FLASH_DK), 0.125


def _note(name, r):
    """worst err / gate of one comparison"""
    return float(r.max()) if r.numel() else 0.0


# ---- references ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,X,Y", [(2, 2, 7, 30), (3, 1, 64, 65), (2, 3, 0, 40)])
def test_flash_reference_matches_sdpa_oracle(B, H, X, Y):
    g = torch.Generator().manual_seed(X + Y)
    L, D = X + Y, H * A.FLASH_DK
    qkv = torch.randn(B, L, 3 * D, generator=g, dtype=torch.float64)
    xl = torch.randint(min(X, 1), X + 1, (B,), generator=g)
    yl = torch.randint(1, Y + 1, (B,), generator=g)
    q, k, v = (t.view(B, L, H, A.FLASH_DK).transpose(1, 2) for t in qkv.split(D, -1))
    keep = torch.rand(B, H, L, L, generator=g) > 0.25
    for kp, p in ((None, 0.0), (keep, 0.25)):
        ds = None if kp is None else kp.double() / (1 - p)
        O, _, _, _ = A.attention_ref(q, k, v, A.flash_visible(xl, yl, X, L)[:, None], SCALE_FLASH, ds)
        want = _sdpa_oracle(qkv, H, X, xl, yl, None if kp is None else kp.double(), p)
        assert (O.transpose(1, 2).reshape(B, L, D) - want).abs().max() <= 1e-12
    assert torch.equal(A.flash_visible(xl, yl, X, L), A.flash_visible_kernel_rule(xl, yl, X, L))


@pytest.mark.parametrize("L", [1, 33, 130])
def test_pad_reference_matches_bert_test_formula(L):
    g = torch.Generator().manual_seed(L)
    B, H = 3, 2
    q, k, v = (torch.randn(B, H, L, 64, generator=g, dtype=torch.float64) for _ in range(3))
    lens = [1, L, max(1, 2 * L // 3)]
    O, _, _, _ = A.attention_ref(q, k, v, A.pad_visible(torch.tensor(lens), L)[:, None], SCALE_64)
    for b in range(B):
        want = ((q[b] @ k[b, :, :lens[b]].transpose(-1, -2)) / 8.0).softmax(-1) @ v[b, :, :lens[b]]
        assert (O[b] - want).abs().max() <= 1e-12                        # every row, padding rows included


@pytest.mark.parametrize("table", ["quarter", "rotary"])
def test_rope_reference_matches_roformer_test_formula(table):
    from oracle import bs_roformer_oracle as O_
    L, H = 33, 2
    q, k, v, gate = A.rope_inputs(2, H, L, 5)
    cs = A.quarter_turn_cs(L) if table == "quarter" else torch.stack(O_.rotary_cos_sin(L), -1)
    got, _ = A.rope_ref(q, k, v, gate, cs, "tf32")
    c, s = cs[:, :, 0].double().repeat_interleave(2, -1), cs[:, :, 1].double().repeat_interleave(2, -1)

    def rot(t):                                                          # test_gpu_bs_roformer._attn_ref
        x = t.unflatten(-1, (-1, 2))
        return t * c + torch.stack((-x[..., 1], x[..., 0]), -1).flatten(-2) * s
    want = torch.softmax(rot(q) @ rot(k).transpose(-1, -2) / 8.0, -1) @ v * torch.sigmoid(gate)[..., None]
    assert (got - want).abs().max() <= 1e-12


def test_philox_and_keep_tensor_layout():
    """keep_tensor of (b, h) is keep_matrix of z = b * H + h with the Philox key words of (seed, offset, stream)"""
    s0, s1, _, _ = A.philox(A.DROP_SEED, 0, 3)
    kt = A.keep_tensor(2, 3, 40, A.DROP_SEED, 0, 3, 0.25)
    assert torch.equal(kt[1, 2], torch.from_numpy(A.keep_matrix(5, 40, s0, s1, 0.25)))
    assert A.drop_threshold(0.1) == int(float(torch.tensor(0.1, dtype=torch.float32)) * 2 ** 32)


# ---- headroom: the emulator stays within the model on every GPU input ----------------------------------------------------
def _flash_readout_inputs(X, Y):
    xl, yl = A.flash_lens(X, Y)
    L = X + Y
    q, k = A.readout_qk(len(xl), L, A.FLASH_DK, 100 * X + Y)
    return q[:, None], k[:, None], xl, yl, A.flash_visible(xl, yl, X, L)


def _assert_readout(got, ref, model, vis, what):
    assert torch.equal(got[~vis.expand_as(got)], torch.zeros_like(got[~vis.expand_as(got)])), what
    return _note(what, A.ratio(got, ref, model))


@pytest.mark.parametrize("mode", MODES)
def test_headroom_flash_readout(mode):
    worst = 0.0
    shapes = [(X, Y) for X in A.FLASH_READOUT_X for Y in A.FLASH_READOUT_Y]
    for X, Y in shapes:
        q, k, xl, yl, vis = _flash_readout_inputs(X, Y)
        ref, model, P = A.readout_ref(q, k, vis, SCALE_FLASH, mode, A.FLASH_TILE)
        assert float(P[vis[:, None]].min()) >= A.PROB_FLOOR, (X, Y)
        got, _ = A.emulate_fwd(q, k, None, vis[:, None], SCALE_FLASH, mode)
        worst = max(worst, _assert_readout(got, ref, model, vis[:, None], f"flash readout {mode}"))
    X, Y, xl, yl = A.FLASH_SHIPPED
    L = X + Y
    q, k = A.readout_qk(2, L, A.FLASH_DK, 7)
    vis = A.flash_visible(torch.tensor(xl), torch.tensor(yl), X, L)
    ref, model, P = A.readout_ref(q[:, None], k[:, None], vis, SCALE_FLASH, mode, A.FLASH_TILE)
    assert float(P[vis[:, None]].min()) >= A.PROB_FLOOR
    got, _ = A.emulate_fwd(q[:, None], k[:, None], None, vis[:, None], SCALE_FLASH, mode)
    worst = max(worst, _assert_readout(got, ref, model, vis[:, None], f"flash readout {mode}"))
    print(f"flash readout {mode}: worst emulated err / gate {worst:.3f}")
    assert worst <= 0.5


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("p", A.DROP_P)
def test_headroom_flash_dropout_readout(mode, p):
    B, X, Y = A.DROP_SHAPE
    L = X + Y
    H = -(-L // A.FLASH_DK)
    xl, yl = torch.tensor([X, X // 2, 1]), torch.tensor([Y, 1, Y - 1])
    q, k = A.readout_qk(B, L, A.FLASH_DK, 11)
    vis = A.flash_visible(xl, yl, X, L)
    keep = A.keep_tensor(B, H, L, A.DROP_SEED, 0, A.DROP_SID, p)
    ds = A.drop_scale(keep, p)
    ref, model, P = A.readout_ref(q[:, None], k[:, None], vis, SCALE_FLASH, mode, A.FLASH_TILE, ds)
    assert float(P[vis[:, None]].min()) >= A.PROB_FLOOR
    got, _ = A.emulate_fwd(q[:, None], k[:, None], None, vis[:, None], SCALE_FLASH, mode, keep, p)
    zero = ~(vis[:, None] & keep)
    assert torch.equal(got == 0, zero)                                    # the zero set is exactly masked or dropped
    r = _note(f"flash dropout readout {mode}", A.ratio(got, ref, model))
    print(f"flash dropout readout p={p} {mode}: worst emulated err / gate {r:.3f}")
    assert r <= 0.5


def _flash_general(case, mode):
    name, B, H, X, Y, pattern, p = case
    L = X + Y
    q, k, v, do, xl, yl = A.flash_general_inputs(B, H, X, Y, pattern, len(name) * 31 + B)
    vis = A.flash_visible(xl, yl, X, L)[:, None]
    keep = A.keep_tensor(B, H, L, A.DROP_SEED, 0, A.DROP_SID, p) if p else None
    ds = None if keep is None else A.drop_scale(keep, p)
    O, lse, P, t = A.attention_ref(q, k, v, vis, SCALE_FLASH, ds)
    bO, Else, Et = A.fwd_model(t, vis, P, lse, v.abs(), mode, A.FLASH_TILE, dscale=ds)
    return dict(q=q, k=k, v=v, do=do, xl=xl, yl=yl, vis=vis, keep=keep, ds=ds, O=O, lse=lse, P=P, t=t, bO=bO, Else=Else,
                Et=Et, p=p, X=X, L=L)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", A.FLASH_GENERAL, ids=[c[0] for c in A.FLASH_GENERAL])
def test_headroom_flash_general(case, mode):
    c = _flash_general(case, mode)
    O, lse = A.emulate_fwd(c["q"], c["k"], c["v"], c["vis"], SCALE_FLASH, mode, c["keep"], c["p"])
    rO = _note(f"flash O {mode}", A.ratio(O, c["O"], c["bO"]))
    rl = _note(f"flash lse {mode}", A.ratio(lse, c["lse"], c["Else"]))
    qr, kr, vr = (c[n].clone().requires_grad_(True) for n in ("q", "k", "v"))
    Or, _, _, _ = A.attention_ref(qr, kr, vr, c["vis"], SCALE_FLASH, c["ds"])
    Or.backward(c["do"])
    bq, bk, bv = A.flash_bwd_model(c["q"], c["k"], c["v"], c["do"], c["vis"], c["P"], c["t"], c["lse"], c["O"], c["bO"],
                                   c["Else"], c["Et"], SCALE_FLASH, mode, c["ds"])
    dq, dk, dv = A.emulate_bwd(c["q"], c["k"], c["v"], c["do"], O, lse, c["vis"], SCALE_FLASH, mode, c["keep"], c["p"])
    rs = [_note(f"flash {n} {mode}", A.ratio(g, w.grad, b)) for n, g, w, b in (("dQ", dq, qr, bq), ("dK", dk, kr, bk), ("dV", dv, vr, bv))]
    print(f"flash {case[0]} {mode}: worst emulated err / gate O {rO:.3f} lse {rl:.3f} dQ {rs[0]:.3f} dK {rs[1]:.3f} dV {rs[2]:.3f}")
    assert max([rO, rl] + rs) <= 0.5


@pytest.mark.parametrize("mode", MODES)
def test_headroom_pad_readout(mode):
    worst = 0.0
    for L in A.PAD_READOUT_L:
        lens = torch.tensor([min(n, L) for n in A.PAD_LENS + (L,)])
        q, k = A.readout_qk(len(lens), L, A.ATTN64_DK, L)
        vis = A.pad_visible(lens, L)
        ref, model, P = A.readout_ref(q[:, None], k[:, None], vis, SCALE_64, mode, A.ATTN64_KEY_TILE)
        assert float(P[vis[:, None]].min()) >= A.PROB_FLOOR
        got, _ = A.emulate_fwd(q[:, None], k[:, None], None, vis[:, None], SCALE_64, mode)
        worst = max(worst, _assert_readout(got, ref, model, vis[:, None], f"attn64 pad readout {mode}"))
    print(f"attn64 pad readout {mode}: worst emulated err / gate {worst:.3f}")
    assert worst <= 0.5


def _rope_emulate(q, k, v, gate, cs, mode):
    """fp32 rotation (as the kernel: Q in registers, A operand; K in shared memory, raw bits = truncation under TF32)"""
    L = q.shape[-2]
    qr, kr = A.rope_rotate(q.float(), cs[:L]).float(), A.rope_rotate(k.float(), cs[:L]).float()
    qe = A.a_operand(qr, mode)
    ke = (kr.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double() if mode == "tf32" else A.a_operand(kr, mode)
    vis = torch.ones(q.shape[:-2] + (L, L), dtype=torch.bool)
    O, _ = A.emulate_fwd(qe, ke, v, vis, SCALE_64, mode)
    return (O.float() * torch.sigmoid(gate.float())[..., None]).double()


@pytest.mark.parametrize("mode", MODES)
def test_headroom_rope(mode):
    from oracle import bs_roformer_oracle as O_
    worst = 0.0
    tables = [(L, A.quarter_turn_cs(L)) for L in A.ROPE_L] + [(A.ROPE_REAL_L, torch.stack(O_.rotary_cos_sin(A.ROPE_REAL_L), -1))]
    for L, cs in tables:
        q, k, v, gate = A.rope_inputs(2, A.ROPE_H, L, L)
        ref, model = A.rope_ref(q, k, v, gate, cs, mode)
        got = _rope_emulate(q, k, v, gate, cs, mode)
        worst = max(worst, _note(f"rope {mode}", A.ratio(got, ref, model)))
    print(f"rope {mode}: worst emulated err / gate {worst:.3f}")
    assert worst <= 0.5


# ---- sensitivity: the element-wise gate rejects every modelled fault ------------------------------------------------------
def _rejects(got, ref, model, vis=None):
    """the element-wise gate fails: a masked / dropped entry is not exactly 0, or some error exceeds its gate or is not
    finite"""
    return bool(A.outside_gate(got, ref, model, None if vis is None else ~vis.expand_as(got)).any())


def test_gate_rejects_non_finite_outputs():
    ref = torch.tensor([1.0, 0.5, 0.25])
    model = torch.full_like(ref, 1e-3)
    assert not _rejects(ref.clone(), ref, model)
    for bad in (float("nan"), float("inf"), -float("inf")):
        got = ref.clone()
        got[1] = bad
        assert _rejects(got, ref, model), bad
        assert A.ratio(got, ref, model)[1] == float("inf")
    assert _rejects(torch.tensor([1.0, 0.5, float("nan")]), torch.tensor([1.0, 0.5, 0.0]), torch.tensor([1e-3, 1e-3, 0.0]),
                    torch.tensor([True, True, False]))


def test_gate_rejects_every_modelled_fault():
    mode = "tf32"
    X, Y = 65, 65
    q, k, xl, yl, vis = _flash_readout_inputs(X, Y)
    L = X + Y
    ref, model, _ = A.readout_ref(q, k, vis, SCALE_FLASH, mode, A.FLASH_TILE)
    good, _ = A.emulate_fwd(q, k, None, vis[:, None], SCALE_FLASH, mode)
    assert not _rejects(good, ref, model, vis[:, None])
    b = int(((xl == X) & (yl == Y)).nonzero()[0])                      # the full item
    faults = {}

    def readout_fault(name, vis_kernel):
        got, _ = A.emulate_fwd(q, k, None, vis_kernel[:, None], SCALE_FLASH, mode)
        faults[name] = (_rejects(got, ref, model, vis[:, None]), A.rel_l2(got, ref) <= TOL_TC)

    v1 = vis.clone(); v1[b, L - 1, 64] = False                         # key 64 (first of a key tile) dropped from the last row
    readout_fault("visible key dropped", v1)
    bh = int(((xl == X // 2) & (yl == Y)).nonzero()[0])
    v2 = vis.clone(); v2[bh, 0, X // 2] = True                         # text padding key xl admitted to row 0
    readout_fault("masked key admitted", v2)
    v3 = A.flash_visible_kernel_rule(xl, yl, X + 1, L)
    assert not torch.equal(v3, vis)
    readout_fault("prefix boundary moved by one", v3)
    qt = 1
    kt = A.flash_key_tiles(qt * A.FLASH_TILE, L, X, int(yl[b])) - 1
    v4 = vis.clone(); v4[b, 64:128, kt * 64:(kt + 1) * 64] = False
    assert bool((vis[b, 64:128, kt * 64:(kt + 1) * 64]).any())
    readout_fault("last key tile of one query tile skipped", v4)
    sw = good.clone(); sw[b, 0, [70, 71]] = good[b, 0, [71, 70]]
    faults["two query rows swapped"] = (_rejects(sw, ref, model, vis[:, None]), A.rel_l2(sw, ref) <= TOL_TC)

    p = A.DROP_P[0]
    B, X, Y = A.DROP_SHAPE
    L = X + Y
    H = -(-L // A.FLASH_DK)
    xl, yl = torch.tensor([X, X // 2, 1]), torch.tensor([Y, 1, Y - 1])
    qd, kd = A.readout_qk(B, L, A.FLASH_DK, 11)
    visd = A.flash_visible(xl, yl, X, L)
    keep = A.keep_tensor(B, H, L, A.DROP_SEED, 0, A.DROP_SID, p)
    refd, modeld, _ = A.readout_ref(qd[:, None], kd[:, None], visd, SCALE_FLASH, mode, A.FLASH_TILE, A.drop_scale(keep, p))
    kf = keep.clone(); kf[0, 1, L - 1, 100] = ~kf[0, 1, L - 1, 100]
    got, _ = A.emulate_fwd(qd[:, None], kd[:, None], None, visd[:, None], SCALE_FLASH, mode, kf, p)
    faults["one keep flag flipped"] = (_rejects(got, refd, modeld, (visd[:, None] & keep)), A.rel_l2(got, refd) <= TOL_TC)

    c = _flash_general(A.FLASH_GENERAL[0], mode)
    _, lse = A.emulate_fwd(c["q"], c["k"], c["v"], c["vis"], SCALE_FLASH, mode)
    lse[0, 0, 5] += 2.0 ** -8
    faults["one row's lse off by 2^-8"] = (_rejects(lse, c["lse"], c["Else"]), A.rel_l2(lse, c["lse"]) <= TOL_TC)

    for name, (rej, l2ok) in faults.items():
        print(f"fault {name!r}: element-wise gate {'rejects' if rej else 'PASSES'}, rel-L2 <= TOL_TC "
              f"{'passes (missed)' if l2ok else 'rejects'}")
    assert all(rej for rej, _ in faults.values()), faults
    assert len(faults) == 7

