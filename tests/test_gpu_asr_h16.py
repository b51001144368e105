"""GPU tests of the 16-bit Linears and of Whisper under a float16 / bfloat16 compute type (`pytest -m gpu`).

Kernels (evk_linear_rows_h16, evk_linear_h16): every output bit for bit against float64 with operands exactly representable
in 16 bits and partial sums exact in fp32; RNE staging of fp32 activations within a per-element accumulation bound (which
truncation of the same inputs breaks); a row's bits independent of the rows beside it.  Model: encoder and teacher-forced
logits against the float64 emulation of 16-bit Linears (tests/whisper_h16_ref.py), beam-search tokens against it, long-form
pooling invariance, the fp32 -> fp16 -> fp32 switch, and `WhisperAsr.recognize` with precision "float16"."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import pin_asr as PIN
from oracle import pin_asr_long as PINL
from oracle import whisper_oracle as O
from tests import whisper_h16_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "asr.pt"), weights_only=False)
GOLD_LONG = torch.load(os.path.join(ROOT, "tests", "golden", "asr_long.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
DTYPES = [torch.float16, torch.bfloat16]
KERNELS = ["linear_rows_h16", "linear_h16"]
SENTINEL = 12345.0
# rel-L2 against the float64 emulation of 16-bit Linears (whisper_h16_ref), measured on an H100 80GB HBM3 (700 W) and
# printed by the test: encoder 4.8e-4 / 4.4e-4 in fp16, 2.2e-3 / 2.1e-3 in bf16; teacher-forced logits 4.6e-4 / 5.7e-4 in
# fp16, 2.9e-3 / 3.3e-3 in bf16 (m80_d2 / m128_d4).  Gates at no more than twice the larger value and below the TF32 path's
# 5e-3 against float64.  The emulation rounds float64 activations where the kernels round fp32 ones; an RNE decision that
# flips between the two moves a product by half a 16-bit ulp, which is why bf16 sits higher.
TOL_ENC = {torch.float16: 1e-3, torch.bfloat16: 4.4e-3}
TOL_LOGITS = {torch.float16: 1.1e-3, torch.bfloat16: 4.5e-3}
# length-normalised beam scores on equal tokens: up to 7.1e-3 relative to the emulation's (m128_d4, bf16)
TOL_SCORE = 1.5e-2


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


@pytest.fixture(scope="module")
def W(ops):
    from easevoice_trainer_b200 import whisper
    return whisper


def run(ops, kernel, x, w, bias=None, act=0, res=None, out=None):
    return getattr(ops, kernel)(x, w, bias, act=act, res=res, out=out)


# ---- exact contractions -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("rows", [1, 5, 17, 70, 128, 300])
def test_exact_contraction(ops, kernel, dtype, rows):
    """x = i / 4 and W = j / 8 with |i|, |j| <= 8 are exact in fp16 and bf16; products are multiples of 1/32 of at most 2,
    so every partial sum over K <= 2000 is exact in fp32 and each output must equal float64.  Operand buffers carry NaN past
    K, the output buffer a sentinel past N; N and K are off the tile sizes (64 columns / 64 K, 128 x 128 / 64 K)."""
    g = torch.Generator().manual_seed(rows)
    for N, K in ((200, 136), (72, 1000), (1300, 1288)):
        xv = torch.randint(-8, 9, (rows, K), generator=g).float() / 4
        wv = torch.randint(-8, 9, (N, K), generator=g).float() / 8
        bias = torch.randint(-16, 17, (N,), generator=g).float() / 32
        res = torch.randint(-64, 65, (rows, N), generator=g).float() / 16
        xbuf = torch.full((rows, K + 9), float("nan"))
        xbuf[:, :K] = xv
        xd = xbuf.to(DEV)[:, :K]
        w = ops.pack_weight_h16(wv.to(DEV), dtype)
        pre = xv.double() @ wv.double().T + bias.double()
        for with_res in (False, True):
            ybuf = torch.full((rows, N + 5), SENTINEL, device=DEV)
            run(ops, kernel, xd, w, bias.to(DEV), res=res.to(DEV) if with_res else None, out=ybuf[:, :N])
            want = pre + res.double() if with_res else pre
            got = ybuf.cpu()
            assert torch.equal(got[:, :N].double(), want), (kernel, N, K, with_res, (got[:, :N].double() - want).abs().max())
            assert torch.all(got[:, N:] == SENTINEL)
        # GELU epilogue: the exact pre-activation through fp32 erf GELU
        y = run(ops, kernel, xd, w, bias.to(DEV), act=ops.ACT_GELU)
        ref = torch.nn.functional.gelu(pre.float().to(DEV))
        assert torch.all((y - ref).abs() <= 2e-6 * ref.abs().clamp(min=1.0))


# ---- rounding -------------------------------------------------------------------------------------------------------------
def midpoints(shape, dtype, g):
    """Positive fp32 values halfway between two neighbouring `dtype` values (RNE rounds half of them up, truncation none)."""
    a = (0.5 + torch.rand(shape, generator=g)).to(dtype)
    b = (a.view(torch.int16) + 1).view(dtype)
    return (a.float() + b.float()) / 2


def truncated(x, dtype):
    """x rounded towards zero to `dtype`."""
    r = x.to(dtype)
    up = r.float().abs() > x.abs()
    return torch.where(up, (r.view(torch.int16) - 1).view(dtype), r).double()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_rounding_at_midpoints(ops, kernel, dtype):
    """Every activation at a 16-bit midpoint, positive weights: each output lies within 2 gamma_K sum|h(x) h(W)| of
    float64(h(x) h(W)) with h = RNE, and the same inputs rounded by truncation land outside that bound."""
    g = torch.Generator().manual_seed(7)
    for rows, N, K in ((5, 136, 256), (300, 200, 520)):
        x = midpoints((rows, K), dtype, g)
        assert torch.all(x.to(dtype).float() != x)
        wv = (0.25 + torch.rand(N, K, generator=g)).to(dtype)
        w = ops.pack_weight_h16(wv.float().to(DEV), dtype)
        y = run(ops, kernel, x.to(DEV), w).double().cpu()
        hw = wv.double()
        want = x.to(dtype).double() @ hw.T
        u = 2.0 ** -24
        bound = 2 * (K * u / (1 - K * u)) * (x.to(dtype).double().abs() @ hw.abs().T)
        err = (y - want).abs()
        print(f"{kernel} {dtype} {rows}x{N}x{K}: max err / bound {(err / bound).max():.3f}")
        assert torch.all(err <= bound)
        trunc = truncated(x, dtype) @ hw.T
        assert torch.all((y - trunc).abs() > bound)


# ---- row invariance -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_row_kernel_row_invariance(ops, dtype):
    """A row's bits are the same at 1, 5, 70 and 300 rows and at any position in the launch, with one K split (N = 4096)
    and with several (N = 1280, K = 5120)."""
    g = torch.Generator().manual_seed(3)
    for N, K in ((1280, 5120), (4096, 1280), (51866 // 8, 1280)):
        x = torch.randn(300, K, generator=g).to(DEV)
        w = ops.pack_weight_h16((torch.randn(N, K, generator=g) / K ** 0.5).to(DEV), dtype)
        b = torch.randn(N, generator=g).to(DEV)
        full = ops.linear_rows_h16(x, w, b)
        for n in (1, 5, 70):
            for r0 in (0, 300 - n):
                assert torch.equal(ops.linear_rows_h16(x[r0:r0 + n], w, b), full[r0:r0 + n]), (N, K, n, r0)


# ---- model level ----------------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def model(W, name, dtype):
    c = GOLD["cases"][name]
    net = W.WhisperModel(c["cfg"], GOLD["gen"]).set_compute_type(dtype)
    sd = PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"])
    net.load_state_dict(sd)
    return net.to(DEV).eval(), c, sd


def oracle_feats(c):
    xs = [PIN.clip(c["seed"] * 10 + i, s) for i, s in enumerate(c["secs"])]
    return torch.stack([O.features(x, c["cfg"]["num_mel_bins"]) for x in xs])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["m80_d2", "m128_d4"])
def test_encoder_and_logits_against_emulation(W, name, dtype):
    net, c, sd = model(W, name, dtype)
    feats = oracle_feats(c)
    enc = net.encode(feats.float().to(DEV))
    ref = R.encode(sd, feats, c["cfg"], dtype)
    e, e32 = rel(enc, ref), rel(enc, O.encode(sd, feats, c["cfg"]))
    toks = c["forced"]
    lg = net.teacher_forced_logits(enc, toks.tolist())
    lref = R.decode_logits(sd, ref, toks, c["cfg"], dtype)
    l, l32 = rel(lg, lref), rel(lg, O.decode_logits(sd, O.encode(sd, feats, c["cfg"]), toks, c["cfg"]))
    print(f"{name} {dtype}: encoder rel-L2 {e:.2e} (fp32 oracle {e32:.2e}), logits {l:.2e} (fp32 oracle {l32:.2e})")
    assert e <= TOL_ENC[dtype] and l <= TOL_LOGITS[dtype]
    # a clip's encoder output is the same alone and batched
    assert torch.equal(net.encode(feats[:1].float().to(DEV))[0], enc[0])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["m80_d2", "m128_d4"])
def test_tokens_against_emulation(W, name, dtype):
    net, c, sd = model(W, name, dtype)
    feats = oracle_feats(c)
    sp = O.special_tokens(GOLD["gen"])
    for lang in ("zh", None):
        got = net.transcribe_features(feats.float().to(DEV), language=lang)
        for i, o in enumerate(got):
            want = R.transcribe_clip(sd, c["cfg"], sp, feats[i], dtype, language=lang)
            assert (o["language"], o["tokens"]) == (want["language"], want["tokens"]), (name, lang, i)
            d = abs(o["score"] - want["score"]) / max(1.0, abs(want["score"]))
            print(f"{name} {dtype} lang={lang} clip {i}: {len(o['tokens'])} tokens equal, score rel diff {d:.1e}")
            assert d <= TOL_SCORE, (o["score"], want["score"])


def test_long_form_pool_invariance(W):
    """Under fp16 each clip of a two-clip pool gets the same tokens and seeks alone and pooled."""
    c = GOLD_LONG["case"]
    net = W.WhisperModel(c["cfg"], GOLD_LONG["gen"]).set_compute_type(torch.float16)
    net.load_state_dict(PINL.make_state_dict(c))
    net = net.to(DEV).eval()
    xs = [PINL.clip(*k) for k in GOLD_LONG["clips"]]
    frames = [x.size // 160 for x in xs]
    L = max(x.size for x in xs)
    wav = torch.zeros(len(xs), L)
    for i, x in enumerate(xs):
        wav[i, :x.size] = torch.from_numpy(x)
    lm = net.features_long(wav.to(DEV), [x.size for x in xs])
    pool = net.transcribe_long(lm, frames, language="de", clips_per_batch=2)
    for i in range(len(xs)):
        alone = net.transcribe_long(lm[i:i + 1, :], frames[i:i + 1], language="de", clips_per_batch=1)[0]
        assert pool[i]["tokens"] == alone["tokens"], i
        assert [w["seek"] for w in pool[i]["windows"]] == [w["seek"] for w in alone["windows"]], i


@pytest.fixture
def packs(monkeypatch):
    """[number of fp32 packs, number of 16-bit packs] so far"""
    from easevoice_trainer_b200 import ops
    n, p32, p16 = [0, 0], ops.pack_weight, ops.pack_weight_h16

    def c32(*a, **k):
        n[0] += 1
        return p32(*a, **k)

    def c16(*a, **k):
        n[1] += 1
        return p16(*a, **k)
    monkeypatch.setattr(ops, "pack_weight", c32)
    monkeypatch.setattr(ops, "pack_weight_h16", c16)
    return n


def test_precision_switch(W, packs):
    """fp32 -> fp16 -> fp32 on one model equals fresh models bit for bit; a second call in the same mode packs nothing; the
    16-bit mode packs only the two convs in fp32."""
    c = GOLD["cases"]["m80_d2"]
    xs = [PIN.clip(c["seed"] * 10 + i, s) for i, s in enumerate(c["secs"])]
    wav = torch.zeros(len(xs), max(x.size for x in xs))
    for i, x in enumerate(xs):
        wav[i, :x.size] = torch.from_numpy(x)
    wav = wav.to(DEV)

    def make(dtype):
        net = W.WhisperModel(c["cfg"], GOLD["gen"]).set_compute_type(dtype)
        net.load_state_dict(PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"]))
        return net.to(DEV).eval()

    def go(net):
        feats = net.features(wav, [x.size for x in xs])
        enc = net.encode(feats)
        return enc.cpu(), net.transcribe_features(feats, language="en", enc=enc)

    net = make(None)
    a = go(net)
    n = list(packs)
    assert torch.equal(go(net)[0], a[0]) and packs == n
    net.set_compute_type(torch.float16)
    b = go(net)
    assert packs[0] - n[0] == 2 and packs[1] > n[1]
    n = list(packs)
    bb = go(net)
    assert packs == n and torch.equal(bb[0], b[0]) and bb[1] == b[1]
    net.set_compute_type(None)
    c2 = go(net)
    fresh16, fresh32 = go(make(torch.float16)), go(make(None))
    assert torch.equal(b[0], fresh16[0]) and b[1] == fresh16[1]
    assert torch.equal(c2[0], fresh32[0]) and c2[1] == fresh32[1] and torch.equal(c2[0], a[0])
    assert not torch.equal(b[0], a[0])


def test_recognize_float16(W, tmp_path):
    """WhisperAsr(..., "float16").recognize writes asr.list lines and trace data of the same shape as "float32"."""
    from scipy.io import wavfile

    from easevoice_trainer_b200 import asr
    from tests.test_gpu_asr import asr_tokenizer
    c = GOLD["cases"]["m80_d2"]
    mdir = tmp_path / "model"
    mdir.mkdir()
    json.dump(dict(c["cfg"]), open(mdir / "config.json", "w"))
    json.dump(GOLD["gen"], open(mdir / "generation_config.json", "w"))
    torch.save(PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"]), mdir / "pytorch_model.bin")
    asr_tokenizer(mdir, GOLD["n_text"])
    files = []
    for i, s in enumerate(c["secs"] + [41.3]):
        f = str(tmp_path / f"clip{i}.wav")
        wavfile.write(f, 16000, PIN.clip(c["seed"] * 10 + i, s).astype(np.float32))
        files.append(f)
    out = {}
    for prec in ("float32", "float16"):
        a = asr.WhisperAsr("large-v3", "zh", prec, model_dir=str(mdir))
        lst, dump = str(tmp_path / f"{prec}.list"), str(tmp_path / f"{prec}.dump")
        res = a.recognize(files, lst, dump)
        assert res.status == "success", res.message
        assert (a.load()[0].compute_type is None) == (prec == "float32")
        out[prec] = (open(lst, encoding="utf-8").read().split("\n"), res.data)
    (l32, d32), (l16, d16) = out["float32"], out["float16"]
    assert len(l16) == len(l32) == len(files) and all(ln.startswith(f + "|zh|") for ln, f in zip(l16, files))
    for f in files:
        assert set(d16[f]) == set(d32[f])
        if "windows" in d32[f]:
            assert [set(w) for w in d16[f]["windows"]] == [set(w) for w in d32[f]["windows"]]
