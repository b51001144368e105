"""CPU rehearsal of tests/cudacore_ref.py: fp32 emulations of the CUDA-core kernels' summation orders stay within the error
model (half the gate) at every element, and modelled faults -- a length mask off by one frame, one lane's dgamma partial
dropped, rstd from the unbiased variance, one chunk missing from the embedding backward, ... -- leave the gate on at least
one element, so the gate is sharp enough to see them."""
import pytest
import torch

from tests import cudacore_ref as R


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def within_model(got, ref, what):
    bad = R.outside_gate(got, ref, factor=1.0)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the model; worst " \
                                f"{float(R.ratio(got, ref).max()) * R.SAFETY:.3f} x model"
    return float(R.ratio(got, ref).max())


def outside(got, ref, what):
    n = int(R.outside_gate(got, ref).sum())
    print(f"fault '{what}': {n} elements outside the gate, worst err/gate {float(R.ratio(got, ref).max()):.3g}")
    assert n > 0, f"fault '{what}' stays inside the gate"


def ln_rows(rows, C, seed, dc=0.0):
    g = _gen(seed)
    x = (torch.randn(rows, C, generator=g) + dc).float()
    x[0] = 0.75                                                      # a constant row: var = 0
    return x


# ---- LayerNorm ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 33, 192, 512, 1024])
@pytest.mark.parametrize("eps", [1e-5, 1e-12])
def test_layernorm_fwd_emulation_within_model(C, eps):
    g = _gen(C)
    for dc in (0.0, 1e3):
        x = ln_rows(12, C, C + int(dc), dc)
        gamma, beta = (1 + 0.1 * torch.randn(C, generator=g)).float(), (0.1 * torch.randn(C, generator=g)).float()
        y, mean, rstd = R.emulate_layernorm_fwd(x, gamma, beta, eps)
        ry, rm, rr = R.layernorm_fwd(R.ln_input(x), gamma, beta, eps, R.ln_row_chain(C))
        within_model(y, ry, f"y C={C} dc={dc}")
        within_model(mean, rm, "mean")
        within_model(rstd, rr, "rstd")


def test_layernorm_fault_unbiased_variance():
    C = 512
    x = ln_rows(16, C, 3)
    gamma, beta = torch.ones(C), torch.zeros(C)
    y, _, _ = R.emulate_layernorm_fwd(x, gamma, beta, 1e-5, unbiased=True)
    ry, _, _ = R.layernorm_fwd(R.ln_input(x), gamma, beta, 1e-5, R.ln_row_chain(C))
    outside(y, ry, "rstd from the unbiased variance")


@pytest.mark.parametrize("rows,C", [(111, 33), (4225, 192)])          # 4225 rows: the first rows_per_block above 8 (rpb = 9)
def test_layernorm_bwd_emulation_within_model(rows, C):
    g = _gen(rows)
    x = ln_rows(rows, C, rows + 1)
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).float()
    dy = torch.randn(rows, C, generator=g).float()
    _, mean, rstd = R.emulate_layernorm_fwd(x, gamma, torch.zeros(C), 1e-5)
    dx, dg, db = R.emulate_layernorm_bwd(x, gamma, mean, rstd, dy)
    rdx, rdg, rdb = R.layernorm_bwd(R.ln_input(x), gamma, mean, rstd, dy, R.ln_row_chain(C), R.ln_param_chain(rows))
    within_model(dx, rdx, "dx")
    within_model(dg, rdg, "dgamma")
    within_model(db, rdb, "dbeta")
    if rows == 4225:
        assert R.ln_bwd_geometry(rows) == (9, 470)
        _, dg_f, _ = R.emulate_layernorm_bwd(x, gamma, mean, rstd, dy, drop_lane=(3, 5, 7))
        outside(dg_f, rdg, "one lane's dgamma partial dropped")


# ---- block_sum / ordered_sum chains --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1000, 600_000])                    # 600,000 > 540,672: a second trip of the g1 grid
def test_reduce_loss_chain_within_model(n):
    g = _gen(n)
    a = torch.randn(n, generator=g).float()
    for kind in (0, 1):
        ref, G = R.reduce_loss(kind, a, None, 0.5)
        terms = ((1.0 - a) * (1.0 - a)).float() if kind == 0 else (a * a).float()
        part = (R.grid_partials(terms, R.G1_CAP) * 0.5).float()
        got = R.ordered_sum(part[:, None], torch.zeros(1))[0]
        within_model(got.reshape(1), R.E(ref.v.reshape(1), (ref.e + R.os_chain(G) * R.U32 * ref.v.abs()).reshape(1)),
                     f"reduce_loss kind {kind} n={n}")


def test_ordered_sum_fault_lost_partial():
    g = _gen(5)
    part = torch.rand(700, 40, generator=g).float()                  # 700 partials: 44 per lane
    ref = R.esum(R.E(part.double()), 0, R.os_chain(700))
    within_model(R.ordered_sum(part, torch.zeros(40)), ref, "ordered_sum")
    lost = part.clone()
    lost[699, 13] = 0.0
    outside(R.ordered_sum(lost, torch.zeros(40)), ref, "ordered_sum loses one partial")


@pytest.mark.parametrize("rows,n", [(1, 1), (63, 31), (65, 33), (20000, 33)])
def test_colsum_chain_within_model(rows, n):
    g = _gen(rows + n)
    x = torch.randn(rows, n, generator=g).float()
    base = torch.randn(n, generator=g).float()
    got = R.emulate_colsum(x, base)
    ref = R.esum(R.E(torch.cat([x, base[None]]).double()), 0, R.colsum_chain(rows, n))
    within_model(got, ref, "colsum accumulate")
    outside(R.emulate_colsum(x), ref, "colsum ignores accumulate = 1")


# ---- cross-entropy, KL, AdamW, embedding ----------------------------------------------------------------------------------
def test_ce_lse_nll_within_model():
    g = _gen(9)
    rows, V = 40, 1025
    logits = (30 * torch.randn(rows, V, generator=g)).float()
    tgt = torch.randint(0, V, (rows,), generator=g)
    lse, nll = R.emulate_ce_fwd(logits, tgt)
    L = R.E(logits.double())
    mx = logits.max(-1).values.double()
    se = R.esum(R.expf(L - R.E(mx[:, None])), -1, R.ln_row_chain(V))
    rlse = R.E(mx) + R.logf(se)
    rnll = rlse - R.E(logits.gather(1, tgt[:, None])[:, 0].double())
    within_model(lse, rlse, "lse")
    within_model(nll, rnll, "nll")
    _, nll_f = R.emulate_ce_fwd(logits, (tgt + 1) % V)
    outside(nll_f, rnll, "nll of the neighbouring class")


def test_kl_within_model_and_mask_fault():
    g = _gen(11)
    B, T, C = 3, 50, 24
    lens = torch.tensor([50, 1, 31])
    zp, lq, mp = (torch.randn(B * T, C, generator=g).float() for _ in range(3))
    lp = (torch.rand(B * T, C, generator=g) * 10 - 7).float()         # logs_p in [-7, 3]: __expf(-2 logs_p) up to e^14
    keep = R.time_mask(B, T, lens)
    terms = R.emulate_kl_terms(zp, lq, mp, lp)
    rt = R.kl_terms(zp, lq, mp, lp)
    within_model(terms, rt, "kl terms")
    n = B * T * C
    ref = R.esum(R.E(torch.where(keep[:, None], rt.v, 0.0), torch.where(keep[:, None], rt.e, 0.0)), (0, 1),
                 R.grid_reduce_chain(n, R.G1_CAP))
    got = R.ordered_sum(R.grid_partials(torch.where(keep[:, None], terms, 0.0), R.G1_CAP)[:, None], torch.zeros(1))
    within_model(got, R.E(ref.v.reshape(1), ref.e.reshape(1)), "kl sum")
    off = R.time_mask(B, T, lens + 1)                                 # the mask one frame too long
    got_f = R.ordered_sum(R.grid_partials(torch.where(off[:, None], terms, 0.0), R.G1_CAP)[:, None], torch.zeros(1))
    outside(got_f, R.E(ref.v.reshape(1), ref.e.reshape(1)), "kl length mask off by one frame")


def test_adamw_three_steps_within_model():
    g = _gen(13)
    n = 5000
    p = torch.randn(n, generator=g).float()
    m, v = torch.zeros(n), torch.zeros(n)
    P, M, Vv = R.E(p.double()), R.E(m.double()), R.E(v.double())
    hp = dict(lr=2e-4, lr_scale=0.5, b1=0.8, b2=0.99, eps=1e-9, wd=0.01, grad_scale=0.25)
    for step in (1, 2, 3):
        gr = torch.randn(n, generator=g).float()
        if step == 2:                                                 # the device step counter not advanced: step 1's bias correction
            p_stale = R.emulate_adamw(p, gr, m, v, step=1, **hp)[0]
        p, m, v, gg = R.emulate_adamw(p, gr, m, v, step=step, **hp)
        P, M, Vv, GG = R.adamw_step(P, gr, M, Vv, step=step, **hp)
        within_model(p, P, f"adamw p step {step}")
        within_model(m, M, f"adamw m step {step}")
        within_model(v, Vv, f"adamw v step {step}")
        within_model(gg, GG, "adamw g^2")
        if step == 2:
            outside(p_stale, P, "adamw with the bias correction of the previous step")


def test_embedding_bwd_fault_missing_chunk():
    g = _gen(17)
    rows, V, C = 1000, 7, 16
    idx = torch.randint(0, V, (rows,), generator=g)
    dy = torch.randn(rows, C, generator=g).float()
    nch = R.cdiv(rows, 256)
    chain = 256 + R.os_chain(nch)
    one = torch.nn.functional.one_hot(idx, V).double()                 # [rows, V]
    ref = R.E(one.T @ dy.double(), chain * R.U32 * (one.T @ dy.double().abs()))
    part = torch.zeros(nch, V * C)
    for k in range(nch):
        acc = torch.zeros(V, C)
        for r in range(k * 256, min(rows, k * 256 + 256)):
            acc[idx[r]] = (acc[idx[r]] + dy[r]).float()
        part[k] = acc.reshape(-1)
    within_model(R.ordered_sum(part, torch.zeros(V * C)).view(V, C), ref, "embedding_bwd")
    outside(R.ordered_sum(part[:-1], torch.zeros(V * C)).view(V, C), ref, "embedding_bwd without its last chunk")


def test_masked_mean_fault_len_off_by_one():
    g = _gen(19)
    T, C = 40, 5
    x = torch.randn(T, C, generator=g).float()
    for n in (1, 17, 40):
        ref = R.esum(R.E(x[:n].double()), 0, R.cdiv(n, 8) + 8) / float(n)
        acc = torch.zeros(8, C)
        for t in range(n):
            acc[t % 8] = acc[t % 8] + x[t]
        s = torch.zeros(C)
        for k in range(8):
            s = s + acc[k]
        within_model((s / n).float(), ref, "masked_mean")
        if n < T:
            outside(((s + x[n]) / (n + 1)).float(), ref, "masked_mean over one frame too many")


def test_error_model_flags_exact_outputs():
    """an output with model 0 (copies, masked zeros) must match bit for bit: the smallest change is outside the gate"""
    ref = R.E(torch.tensor([0.0, 1.5, -2.0]))
    assert not bool(R.outside_gate(torch.tensor([0.0, 1.5, -2.0]), ref).any())
    assert bool(R.outside_gate(torch.tensor([0.0, float(torch.nextafter(torch.tensor(1.5), torch.tensor(2.0))), -2.0]), ref).any())
    assert bool(R.outside_gate(torch.tensor([float("nan"), 1.5, -2.0]), ref).any())
