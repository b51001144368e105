"""CPU tests: the C ABI (header <-> shared library), and the host-side logic around the kernels."""
import ctypes
import io
import json
import os
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
    # 7 pointers + 9 int64 + 19 int32 + float + int32[48] + (pointer, uint64, float) of the fused-dropout request, padded to 8 bytes
    expect = 7 * 8 + 9 * 8 + 19 * 4 + 4 + 48 * 4 + 8 + 8 + 4
    assert ctypes.sizeof(lib.GconvDesc) == (expect + 7) // 8 * 8
    assert lib.GconvDesc.off.offset == 7 * 8 + 9 * 8 + 19 * 4 + 4
    assert lib.GconvDesc.drop_rng.offset == 400 and lib.GconvDesc.drop_sid.offset == 408 and lib.GconvDesc.drop_p.offset == 416
    assert lib.load().evk_gconv_desc_size() == ctypes.sizeof(lib.GconvDesc)          # the compiled header agrees with the ctypes mirror


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


def test_dgrad_phase_plan_covers_every_tap_exactly_once():
    from easevoice_trainer_b200.ops import dgrad_phase_plan
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
        for u0, Ju, q0, nq, off in dgrad_phase_plan(Q, s, pad, dil, Tin):
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
