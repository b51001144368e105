"""CPU tests: the C ABI (header <-> shared library), and the host-side logic around the kernels."""
import ctypes
import io
import json
import os
import subprocess
from contextlib import redirect_stdout

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_symbol_declared_in_header():
    import __graft_entry__ as g
    g.build()
    from easevoice_trainer_b200 import lib
    protos = lib.parse_header()
    assert len(protos) >= 55
    L = lib.load()                                  # raises AttributeError on any declared-but-missing symbol
    for name in protos:
        assert hasattr(L, name), name
    assert L.evk_version() == 100


def test_descriptor_struct_layout():
    from easevoice_trainer_b200 import lib
    # 7 pointers + 9 int64 + 19 int32 + float + int32[48] + (pointer, uint64, float) of the dropout request + int32
    # no_phase_split + int32 no_grad, padded to 8 bytes
    expect = 7 * 8 + 9 * 8 + 19 * 4 + 4 + 48 * 4 + 8 + 8 + 4 + 4 + 4
    assert ctypes.sizeof(lib.GconvDesc) == (expect + 7) // 8 * 8 == 432
    assert lib.GconvDesc.off.offset == 7 * 8 + 9 * 8 + 19 * 4 + 4
    assert lib.GconvDesc.drop_rng.offset == 400 and lib.GconvDesc.drop_sid.offset == 408 and lib.GconvDesc.drop_p.offset == 416
    assert lib.GconvDesc.no_phase_split.offset == 420
    assert lib.GconvDesc.no_grad.offset == 424
    assert lib.load().evk_gconv_desc_size() == ctypes.sizeof(lib.GconvDesc)          # the compiled header agrees with the ctypes mirror


def test_run_desc_hook_keeps_the_transposed_dy(monkeypatch):
    """Timing hooks (bench.py --config 5) wrap ops._run_desc(fn, d) with two arguments: the weight gradient's transposed dY
    and the data gradient's transposed weight travel on the descriptor, so a wrapped launch still reaches evk_gconv_wgrad /
    evk_gconv_dgrad with them."""
    from easevoice_trainer_b200 import ops
    seen = []

    class FakeLib:
        def evk_gconv_wgrad(self, d, dyt, ld_dyt, stream):
            seen.append((dyt, ld_dyt))
            return 0

        def evk_gconv_dgrad(self, d, wt, ld_wt, stream):
            seen.append(("dgrad", wt, ld_wt))
            return 0

        def evk_gconv_fwd(self, d, stream):
            seen.append(())
            return 0

    monkeypatch.setattr(ops, "_lib", FakeLib)
    monkeypatch.setattr(ops, "_st", lambda: None)
    orig = ops._run_desc

    def hook(fn, d):
        orig(fn, d)

    d = ops._desc(Z=1, C=4, N=4, Q=1, J=1, P=1)
    d.dyt, d.ld_dyt = ctypes.c_void_p(4096), 32
    hook("evk_gconv_wgrad", d)
    hook("evk_gconv_wgrad", ops._desc(Z=1, C=4, N=4, Q=1, J=1, P=1))
    hook("evk_gconv_fwd", d)
    dd = ops._desc(Z=1, C=4, N=4, Q=1, J=1, P=1)
    dd.wt, dd.ld_wt = ctypes.c_void_p(8192), 12
    hook("evk_gconv_dgrad", dd)
    hook("evk_gconv_dgrad", ops._desc(Z=1, C=4, N=4, Q=1, J=1, P=1))
    assert seen[0][0].value == 4096 and seen[0][1] == 32
    assert seen[1] == (None, 0) and seen[2] == ()
    assert seen[3][0] == "dgrad" and seen[3][1].value == 8192 and seen[3][2] == 12
    assert seen[4] == ("dgrad", None, 0)


def test_pack_job_struct_layout():
    from easevoice_trainer_b200 import lib
    # 7 pointers + 8 int32 (D0, D1, Q, lda, D0p, ldb, D1p, row0)
    assert ctypes.sizeof(lib.PackJob) == 7 * 8 + 8 * 4
    assert lib.PackJob.D0.offset == 56 and lib.PackJob.row0.offset == 84
    assert lib.load().evk_pack_job_size() == ctypes.sizeof(lib.PackJob)


def test_no_cpu_fallback():
    """Without an H100 the product path must fail loudly, never silently compute on the CPU."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from easevoice_trainer_b200 import lib, ops
    with pytest.raises(RuntimeError, match="no CPU fallback|evk_init failed"):
        lib.init()
    with pytest.raises(Exception):
        ops.lrelu(torch.zeros(2, 3, 4), 0.1)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "easevoice-trainer_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_state_dict_contract():
    from easevoice_trainer_b200 import models
    from oracle import s2_oracle
    g = models.SynthesizerTrn(1025, 32, n_speakers=300, **s2_oracle.S2_MODEL)
    d = models.MultiPeriodDiscriminator(False)
    for net, spec in ((g, s2_oracle.generator_param_spec()), (d, s2_oracle.discriminator_param_spec())):
        sd = net.state_dict()
        assert set(sd) == set(spec)
        assert all(tuple(sd[k].shape) == tuple(spec[k]) for k in spec)
    assert sum(p.numel() for p in g.parameters()) == 51_310_080
    # weight_norm init: g = ||v||
    v, gg = g.P("dec.ups.0.weight_v"), g.P("dec.ups.0.weight_g")
    assert torch.allclose(gg.flatten(), v.flatten(1).norm(dim=1))
    assert float(g.P("flow.flows.0.post.weight").abs().max()) == 0.0


def test_generator_lr_groups():
    from easevoice_trainer_b200 import models
    from easevoice_trainer_b200.train.s2_step import g_param_groups
    from oracle import s2_oracle
    g = models.SynthesizerTrn(1025, 32, n_speakers=300, **s2_oracle.S2_MODEL)
    groups = g_param_groups(g, 0.4)
    assert [s for s, _ in groups] == [1.0, 0.4, 0.4, 0.4]
    names = [n for _, ns in groups for n in ns]
    assert sorted(names) == sorted(n for n, _ in g.named_parameters())
    assert all(n.startswith("enc_p.encoder_text.") for n in groups[2][1]) and len(groups[1][1]) == 1


_PLAN_SHIM = r"""
#include "dgrad_plan.h"
// the conv's taps at off[q] = q*dil - pad; out = {u0, J, q0, nq, off[0..nq)}
extern "C" int dgrad_phase_c(int Q, int s, int pad, int dil, int Tin, int rho, int* out) {
  int off[EVK_MAX_TAPS];
  for (int q = 0; q < Q; ++q) off[q] = q * dil - pad;
  evk::DgradPhase ph;
  if (!evk::dgrad_phase(off, Q, s, Tin, rho, ph)) return 0;
  out[0] = ph.u0; out[1] = ph.J; out[2] = ph.q0; out[3] = ph.nq;
  for (int k = 0; k < ph.nq; ++k) out[4 + k] = ph.off[k];
  return 1;
}
"""


@pytest.fixture(scope="module")
def dgrad_plan(tmp_path_factory):
    """the library's polyphase plan of a conv data gradient (csrc/dgrad_plan.h) compiled for the host"""
    d = tmp_path_factory.mktemp("dgrad_plan")
    (d / "shim.cpp").write_text(_PLAN_SHIM)
    so = str(d / "libdgrad_plan.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "easevoice-trainer_b200", "csrc"), "-o", so,
                    str(d / "shim.cpp")], check=True)
    fn = ctypes.CDLL(so).dgrad_phase_c
    fn.argtypes = [ctypes.c_int] * 6 + [ctypes.POINTER(ctypes.c_int)]

    def plan(Q, s, pad, dil, Tin):
        """-> [(u0, Ju, q0, nq, off)] over the tap residues, as evk_gconv_dgrad launches them"""
        out, phases = (ctypes.c_int * 64)(), []
        for rho in range(s):
            if fn(Q, s, pad, dil, Tin, rho, out):
                phases.append((out[0], out[1], out[2], out[3], list(out[4:4 + out[3]])))
        return phases
    return plan


def test_library_dgrad_plan_covers_every_tap_exactly_once(dgrad_plan):
    for Q, s, pad, dil, Tin in [(5, 3, 2, 1, 37), (41, 4, 20, 1, 100), (16, 10, 3, 1, 64), (11, 1, 25, 5, 50), (2, 2, 0, 1, 9),
                                (15, 1, 7, 1, 33), (8, 2, 3, 1, 21)]:
        J = (Tin + 2 * pad - dil * (Q - 1) - 1) // s + 1 if s > 1 or True else 0
        want = {}
        for j in range(max(J, 0)):
            for q in range(Q):
                u = j * s - pad + q * dil
                if 0 <= u < Tin:
                    want.setdefault(u, set()).add((q, j))
        got = {}
        for u0, Ju, q0, nq, off in dgrad_plan(Q, s, pad, dil, Tin):
            for jj in range(Ju):
                u = u0 + s * jj
                assert 0 <= u < Tin
                for k in range(nq):
                    q, j = q0 + k * s, jj + off[k]
                    if 0 <= j < J:
                        assert (q, j) not in got.get(u, set())
                        got.setdefault(u, set()).add((q, j))
        assert got == want, (Q, s, pad, dil, Tin)


def test_stdout_protocol_and_checkpoint_layout(tmp_path):
    from easevoice_trainer_b200.utils import ckpt
    from easevoice_trainer_b200.utils.connector import MultiProcessOutputConnector
    from easevoice_trainer_b200.utils.response import EaseVoiceResponse, ResponseStatus
    buf = io.StringIO()
    with redirect_stdout(buf):
        c = MultiProcessOutputConnector()
        c.write_loss(10, 1.5, {"loss/g/total": 1.5, "loss/d/total": 2.0, "learning_rate": 1e-4})
        c.write_response(EaseVoiceResponse(ResponseStatus.SUCCESS, "Finish train sovits", data={"model_path": "x"}))
    l1, l2 = buf.getvalue().strip().split("\n")
    assert l1.startswith("loss-of-easevoice ") and json.loads(l1.split(" ", 1)[1])["step"] == 10
    assert l2.startswith("response-of-easevoice ") and json.loads(l2.split(" ", 1)[1]) == {
        "status": "success", "message": "Finish train sovits", "data": {"model_path": "x"}, "uuid": None}

    class Opt:
        def state_dict(self):
            return {"state": {}, "param_groups": []}

        def load_state_dict(self, sd):
            self.loaded = sd
    net = torch.nn.Linear(3, 2)
    os.chdir(tmp_path)
    path = str(tmp_path / "G_latest.pth")
    ckpt.save_checkpoint(net, Opt(), 1e-4, 7, path)
    saved = torch.load(path)
    assert set(saved) == {"model", "iteration", "optimizer", "learning_rate"} and saved["iteration"] == 7
    net2 = torch.nn.Linear(3, 2)
    _, _, lr, it = ckpt.load_checkpoint(path, net2, Opt())
    assert it == 7 and torch.equal(net2.weight, net.weight)
    assert ckpt.latest_checkpoint_path(str(tmp_path), "G_*.pth") == path
    sd = {"enc_q.pre.weight": torch.ones(2), "dec.conv_pre.weight": torch.ones(2)}
    out = ckpt.export_weights(sd, {"data": {}, "train": {}, "model": {}}, "m_e1_s2", 1, 2, str(tmp_path))
    ex = torch.load(out)
    assert list(ex["weight"]) == ["dec.conv_pre.weight"] and ex["weight"]["dec.conv_pre.weight"].dtype == torch.float16
    assert ex["info"] == "1epoch_2iteration" and "config" in ex


def test_collate_and_bucket_sampler():
    from easevoice_trainer_b200.train import data
    items = [(torch.randn(1, 768, n), torch.randn(1, n * 640), torch.arange(5 + n % 3)) for n in (40, 33, 51)]
    b = data.TextAudioSpeakerCollate(640)(items)
    assert b["lengths"].tolist() == [51, 40, 33] and b["ssl"].shape == (3, 768, 52) and b["wav"].shape == (3, 1, 52 * 640)
    lens = [40, 50, 310, 320, 330, 450, 35, 33] * 10
    seen = []
    for r in range(2):
        s = data.DistributedBucketSampler(lens, 4, [32, 300, 400, 500], 2, r)
        s.set_epoch(3)
        bs = list(iter(s))
        assert len(bs) == len(s) and all(len(x) == 4 for x in bs)
        for batch in bs:                                     # one bucket per batch
            ks = {next(i for i in range(3) if [32, 300, 400, 500][i] < lens[k] <= [32, 300, 400, 500][i + 1]) for k in batch}
            assert len(ks) == 1
        seen.append({k for x in bs for k in x})
    assert seen[0] | seen[1] == set(range(len(lens)))


def test_gpt_state_dict_contract_and_step_schedule():
    """Text2SemanticDecoder mirror: reference state_dict keys/shapes (Lightning adds "model."); training_step schedule
    (t2s_lightning_module.py:52-56): update when batch_idx > 0 and batch_idx % 4 == 0."""
    from oracle import gpt_oracle
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder, sine_table, make_reject_y
    from easevoice_trainer_b200.configs import GPT_MODEL
    m = dict(GPT_MODEL, n_layer=2)
    net = Text2SemanticDecoder({"model": m})
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == gpt_oracle.gpt_param_spec(m)
    assert all(v.dtype == torch.float32 for v in net.state_dict().values())
    assert torch.equal(sine_table(40, 512), gpt_oracle.sine_pe(40, 512))
    y = torch.randint(0, 1024, (3, 20)); yl = torch.tensor([20, 11, 7])
    y_in, tg = net.make_targets(y, yl)
    assert torch.equal(tg[:, :-1], y_in[:, 1:]) and (tg[1, 11:] == 1024).all() and (tg[0, -1] == 1024) and torch.equal(y_in[2, :7], y[2, :7]) \
        and torch.equal(tg[2, :6], y[2, 1:7]) and tg[2, 6] == 1024 and (y_in[2, 7:] == 1024).all()
    ry, rl = make_reject_y(y, yl, torch.Generator().manual_seed(0))
    assert ry.shape[1] == int(rl.max()) and (rl >= 20).all()
    from easevoice_trainer_b200.train.gpt_step import GptStep
    sched = []
    class _S:                                   # only the schedule logic is exercised on CPU
        ACCUM = GptStep.ACCUM
    s = _S()
    for i in range(10):
        s.batch_idx = i
        sched.append(GptStep.wants_step(s))
    assert [i for i, v in enumerate(sched) if v] == [4, 8]


def test_gpt_dataset_collate_and_sampler(tmp_path):
    from easevoice_trainer_b200.train import data_gpt
    table = {f"p{i}": i for i in range(732)}
    g = torch.Generator().manual_seed(0)
    (tmp_path / "3-bert").mkdir()
    with open(tmp_path / "2-name2text.txt", "w") as f2, open(tmp_path / "6-name2semantic.tsv", "w") as f6:
        f6.write("item_name\tsemantic_audio\n")
        for i in range(30):
            nph = 10 + i
            nsem = nph * 25 // 8 if i != 7 else nph * 25 * 2          # utt7: 0.5 phonemes/s -> filtered (min_ps_ratio 3)
            f2.write(f"u{i}\t" + " ".join(f"p{(3 * i + k) % 732}" for k in range(nph)) + "\tw\tt\n")
            f6.write(f"u{i}\t" + " ".join(str((7 * i + k) % 1024) for k in range(nsem)) + "\n")
            if i % 3 == 0:
                torch.save(torch.randn(1024, nph, generator=g), tmp_path / "3-bert" / f"u{i}.pt")
    ds = data_gpt.Text2SemanticDataset(str(tmp_path / "2-name2text.txt"), str(tmp_path / "6-name2semantic.tsv"), max_sec=54, phoneme_table=table)
    assert len(ds) == 29 * 3 and "u7" not in ds.item_names        # < 100 items are replicated max(2, int(100 / n)) times
    b = ds.collate([ds[0], ds[5], ds[9]])
    X, Y = int(b["phoneme_ids_len"].max()), int(b["semantic_ids_len"].max())
    assert b["phoneme_ids"].shape == (3, X) and b["semantic_ids"].shape == (3, Y) and b["bert_feature"].shape == (3, 1024, X)
    assert b["phoneme_ids"].dtype == torch.int64 and b["semantic_ids"].dtype == torch.int64
    i = int(b["semantic_ids_len"].argmin())
    assert (b["semantic_ids"][i, b["semantic_ids_len"][i]:] == 1024).all() and (b["phoneme_ids"][i, b["phoneme_ids_len"][i]:] == 0).all()
    assert float(b["bert_feature"][1].abs().sum()) == 0.0 or ds.item_names[5] in ("u0", "u3", "u6", "u9", "u12", "u15", "u18", "u21", "u24", "u27")
    parts = []
    for r in range(2):
        sp = data_gpt.DistributedBucketSampler(ds, 2, r, batch_size=4)
        sp.set_epoch(3)
        parts.append(list(sp))
    assert len(parts[0]) == len(parts[1]) == (len(ds) + 1) // 2
    assert set(parts[0]) | set(parts[1]) == set(range(len(ds)))    # every sample visited; ranks take alternating slots
    sp0 = data_gpt.DistributedBucketSampler(ds, 2, 0, batch_size=4); sp0.set_epoch(3)
    assert list(sp0) == parts[0]                                   # deterministic in (seed, epoch)


def test_bench_reference_arm_prints_one_json_line():
    """`bench.py --impl reference` (the CPU arm the driver runs next to ours) must emit exactly one JSON line on stdout with the
    contract keys, without touching a GPU or the reference checkout."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--cpu-batch", "1"], capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["n_gpus"] == 1
    assert d["metric"].startswith("s2 SoVITS+HiFiGAN") and d["unit"] == "audio-s/s" and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["e2e"]["h2d_bytes_per_step"] == 0


_GEMV_SHIM = r"""
#include "gemv_route.h"
extern "C" int gemv_route_c(const evk_gconv_desc* d) { return evk::gconv_fwd_gemv(d) ? 1 : 0; }
"""


def test_library_gemv_route_keeps_the_python_rule(tmp_path):
    """Route 0 of evk_gconv_fwd (csrc/gemv_route.h, compiled for the host) takes exactly the Linear launches that ops.linear
    sent to evk_gemv_rows before the rule moved into the library, for descriptors as ops.linear builds them."""
    from easevoice_trainer_b200 import lib, ops
    (tmp_path / "shim.cpp").write_text(_GEMV_SHIM)
    so = str(tmp_path / "libgemv_route.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "easevoice-trainer_b200", "csrc"), "-o", so,
                    str(tmp_path / "shim.cpp")], check=True)
    route = ctypes.CDLL(so).gemv_route_c
    route.argtypes = [ctypes.POINTER(lib.GconvDesc)]

    def python_rule(rows, C, ldw, act, no_grad, res, out_len, in_len, drop):
        """ops.linear's skinny-row condition as it stood before the move (packed weights: Q == 1, ldw % 4 == 0, aligned)"""
        pow2 = 1 if rows == 1 else 2 if rows == 2 else 4
        return (no_grad and not res and not out_len and not in_len and not drop and act in (ops.ACT_NONE, ops.ACT_RELU, ops.ACT_LRELU)
                and 1 <= rows <= 4 and C >= 4 and C % 4 == 0 and C <= ldw and pow2 * C <= 10240)

    n = taken = 0
    for B, T in ((1, 1), (1, 2), (2, 1), (1, 3), (3, 1), (2, 2), (1, 4), (4, 1), (1, 5), (5, 1), (2, 3), (1, 64)):
        rows = B * T
        for C in (1, 2, 3, 4, 6, 8, 510, 512, 2048, 2556, 2560, 2564, 3412, 3416, 5120, 5124, 10240, 10244):
            for ldw in sorted({C, C + 2, C + 4, (C + 3) // 4 * 4, C - 4 if C > 4 else C}):
                if ldw % 4:
                    continue                                   # packed weights: lda is a multiple of 4 (or < 4 with C < 4)
                for act in (ops.ACT_NONE, ops.ACT_RELU, ops.ACT_LRELU, ops.ACT_TANH, ops.ACT_GELU):
                    for flags in range(32):
                        no_grad, res, out_len, in_len, drop = [(flags >> k) & 1 for k in range(5)]
                        if drop and act != ops.ACT_RELU:
                            continue                           # the library rejects these launches before routing
                        N = 96
                        # as _fwd_like builds it: x [B, T, C] dense with pitch C, y [B, T, N], res [B, T, N]
                        d = ops._desc(x=0x10000, w=0x20000, y=0x30000, res=0x40000 if res else 0, out_len=0x50000 if out_len else 0,
                                      in_len=0x60000 if in_len else 0, x_sb=T * C, w_sq=N * ldw, y_sb=T * N, r_sb=T * N if res else 0,
                                      ldx=C, ldw=ldw, ldy=N, ldr=N if res else 0, Z=B, C=C, N=N, Q=1, Tin=T, J=T, P=1, is_=1,
                                      os_=1, Tout=T, act=act, off=[0], no_grad=no_grad)
                        if drop:
                            d.drop_rng, d.drop_sid, d.drop_p = 0x70000, 1, 0.1
                        want = python_rule(rows, C, ldw, act, no_grad, res, out_len, in_len, drop)
                        assert bool(route(ctypes.byref(d))) == want, (B, T, C, ldw, act, flags)
                        n += 1
                        taken += want
    assert n > 10000 and taken > 100, (n, taken)
    # what the Python rule never saw: a misaligned or unevenly pitched weight, and rows that are not evenly spaced
    d = ops._desc(x=0x10000, w=0x20004, y=0x30000, x_sb=2 * 64, w_sq=96 * 64, y_sb=2 * 96, ldx=64, ldw=64, ldy=96, Z=2, C=64, N=96, Q=1,
                  Tin=2, J=2, P=1, is_=1, os_=1, Tout=2, off=[0], no_grad=1)
    assert not route(ctypes.byref(d))
    d.w = 0x20000
    assert route(ctypes.byref(d))
    d.x_sb = 3 * 64
    assert not route(ctypes.byref(d))
