"""GPU parity tests proper (`pytest -m gpu`): CUDA path (through the C ABI) vs the CPU oracle + reference goldens."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GROUPS = ["conv", "conv_transpose", "elementwise", "attention", "vq_losses_optim", "mel", "s2_small", "s2_ragged", "api",
          "gpt_kernels", "scaled_adam", "gpt_small", "gpt_ragged", "gpt_dpo_trainer", "gemm_tma", "vocoder_cfg5",
          "s2_cfg3", "s2_cfg3r", "gpt_cfg2", "sovits_train_e2e", "stft_mrstft", "fused_dropout", "side_streams", "normalize_token", "decode", "infer_panel", "hubert"]


@pytest.fixture(scope="module")
def evk():
    from easevoice_trainer_b200 import lib
    L = lib.init()          # raises loudly if libevk_sm90.so or the H100 is missing: there is no fallback path
    L.evk_set_precise(0)
    return L


@pytest.mark.parametrize("idx", range(len(GROUPS)), ids=GROUPS)
def test_group(evk, idx):
    from tests import checks
    rows = checks.ALL[idx]()
    torch.cuda.synchronize()
    bad = [(n, e, t) for n, e, t in rows if not (e == e and e <= t)]
    assert not bad, "\n".join(f"{n}: err={e:.3e} > tol={t:.1e}" for n, e, t in bad)


def test_precise_mode_tightens_conv(evk):
    """3xTF32 mode must agree with the fp32 oracle ~100x tighter than plain TF32 (proves the error is rounding, not indexing)."""
    from tests import checks
    evk.evk_set_precise(1)
    checks.PRECISE_MODE[0] = True
    try:
        rows = checks.check_conv() + checks.check_conv_transpose()
    finally:
        evk.evk_set_precise(0)
        checks.PRECISE_MODE[0] = False
    # linear paths: <= 1e-4; paths through (leaky-)ReLU: <= 5e-3 (fp32-level derivative flips only)
    bad = [(n, e) for n, e, t in rows if not (e == e and e <= min(t, 5e-3))]
    assert not bad, "\n".join(f"{n}: err={e:.3e}" for n, e in bad)
    lin = [e for n, e, t in rows if " y" in n[-3:]]
    assert max(lin) <= 1e-4, max(lin)


def test_precise_mode_tightens_gpt(evk):
    """3xTF32 in the fused attention + linear kernels: attention agrees with the fp32 oracle at fp32 level, and the
    assembled GPT gradient error collapses (what remains are ReLU-kink flips)."""
    from tests import checks
    evk.evk_set_precise(1)
    checks.PRECISE_MODE[0] = True
    try:
        rows = checks.check_gpt_kernels()
        g_rows = checks.check_gpt("ragged")
    finally:
        evk.evk_set_precise(0)
        checks.PRECISE_MODE[0] = False
    flash = [(n, e) for n, e, t in rows if n.startswith("flash") and "drop-fraction" not in n]
    bad = [(n, e) for n, e in flash if not e <= 2e-5]
    assert not bad, bad
    bad = [(n, e, t) for n, e, t in g_rows if not (e == e and e <= t)]
    assert not bad, bad
    glob = [e for n, e, t in g_rows if "grads global" in n][0]
    assert glob <= 5e-3, glob


def test_sovits_train_two_ranks_ragged_shapes(evk):
    """ADVICE r1 (high): ranks whose batches have different lengths must still capture / replay / all-reduce in lock-step
    (shapes agreed over the gloo side group, no collectives in warm-up).  Needs 2 GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from tests import checks
    rows = checks.check_sovits_train_e2e(gpu_ids="0,1")
    bad = [(n, e, t) for n, e, t in rows if not (e == e and e <= t)]
    assert not bad, bad


def test_s2_steps_are_reproducible(evk):
    """Two runs of three stage-2 optimisation steps from the same weights, batch and RNG seed give bit-identical losses and
    parameters: every reduction across blocks adds its partial sums in a fixed order."""
    from tests import checks
    from easevoice_trainer_b200 import ops
    from easevoice_trainer_b200.train import s2_step
    from oracle import s2_oracle

    def run():
        net_g, net_d, _, _ = checks._load_models()
        net_g.train(); net_d.train()
        ops.manual_seed(7)
        st = s2_step.S2Step(net_g, net_d, dict(s2_oracle.S2_TRAIN), dict(s2_oracle.S2_DATA))
        host = s2_step.synthetic_batch(4, 160, 40, "cuda", seed=3)
        batch = s2_step.to_device_batch(host, torch.device("cuda", 0), st.bank)
        losses = [{k: float(v) for k, v in st.step(batch).items()} for _ in range(3)]
        torch.cuda.synchronize()
        params = torch.cat([p.detach().reshape(-1) for p in list(net_g.parameters()) + list(net_d.parameters())]).cpu()
        return losses, params

    la, pa = run()
    lb, pb = run()
    assert la == lb, (la, lb)
    assert torch.equal(pa, pb), float((pa - pb).abs().max())
