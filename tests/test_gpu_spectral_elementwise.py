"""Every output of the spectral kernels -- the warp-per-frame log-mel front end (evk_mel_fwd), the general STFT (evk_stft_fwd),
their adjoint (evk_mel_bwd / evk_stft_bwd), spec_to_mel, the inverse STFT (evk_istft) and the complex L1 loss (evk_cplx_l1) --
against float64, element for element, with the per-element bound of tests/spectral_ref.py (gate = SAFETY x model).

The C entry points are called directly so that rows can sit in pitched buffers (ldw > L): the samples past each row's own
length and the pitch padding hold NaN, so a read outside the row poisons an output.  Outputs are NaN-prefilled and their pitch
padding holds SENTINEL; dwav and the loss start from a random base that the reference adds.  Every case runs twice and must
give the same bits.  Exact by construction, and checked bit for bit: frames past a row's own count (|X| = 0, X = 0, log-mel =
logf(1e-5f)), the samples of dwav at n >= Lrow, pitch padding, dwav of a silent row, a zero gradient where a == b, and
spec_to_mel of a kernel's own |X| against its fused log-mel (the same fmaf order and the same logf).
The 50 cases take about 10 s on an H100 80GB HBM3 (700 W power limit).
"""
import pytest
import torch

from easevoice_trainer_b200.mel_processing import slaney_filterbank
from tests import cudacore_ref as R
from tests import spectral_ref as S
from tests.test_gpu_cudacore_elementwise import DEV, NAN, SENTINEL, P, _gen, body, check, output, twice, WORST

pytestmark = pytest.mark.gpu
MINE = set()


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init()
    try:
        yield ops
    finally:
        lib.init().evk_set_mel_variant(1)
        for k in sorted(MINE):
            print(f"worst err / gate  {k}: {WORST[k]:.3f}")


def chk(got, ref, what):
    MINE.add(what.split(" ")[0])
    return check(got, ref, what)


_banks = {}


def bank(ops, sr, N, n_mels):
    key = (sr, N, n_mels)
    if key not in _banks:
        fb = slaney_filterbank(sr, N, n_mels)
        _banks[key] = (ops.MelBank(fb, DEV), torch.as_tensor(fb).double())
    return _banks[key]


def wave(B, L, ldw, lens, seed, silent=()):
    """x [B, L] (uniform noise; rows in `silent` all zero) and its pitched buffer: NaN past each row's own length"""
    x = torch.rand(B, L, generator=_gen(seed)) - 0.5
    buf = torch.full((B, ldw), NAN)
    for b in range(B):
        if b in silent:
            x[b] = 0
        Lr = L if lens is None else min(lens[b], L)
        buf[b, :Lr] = x[b, :Lr]
    return x, buf


_LOGCLIP = {}


def logf_clip():
    """the device's logf(1e-5f): what a frame past a row's own count holds"""
    if not _LOGCLIP:
        _LOGCLIP[0] = float(torch.log(torch.tensor([S.CLIP], device=DEV)).cpu()[0])
    return _LOGCLIP[0]


def n_frames(L, N, hop, pad):
    return (L + 2 * pad - N) // hop + 1


def run_fwd(ops, kind, buf, lens_d, B, L, ldw, N, hop, win, pad, T, bk, n_mels, want):
    NB = N // 2 + 1
    spec = output(B * T, NB, NB + 3) if "spec" in want else None
    mel = output(B * T, n_mels, n_mels + 2) if "mel" in want else None
    cplx = torch.full((B * T, NB, 2), NAN, device=DEV) if "cplx" in want else None
    wd = buf.to(DEV)
    if kind == "mel":
        ops._call("evk_mel_fwd", P(wd), P(lens_d), B, L, ldw, hop, n_mels, P(bk.ptr), P(bk.idx), P(bk.val), P(spec), NB + 3, P(mel),
                  n_mels + 2, P(cplx))
    else:
        ops._call("evk_stft_fwd", P(wd), P(lens_d), B, L, ldw, N, hop, win, pad, T, S.EPS, P(cplx), P(spec), NB + 3, n_mels, P(bk.ptr),
                  P(bk.idx), P(bk.val), S.CLIP, P(mel), n_mels + 2)
    return spec, mel, cplx


def fwd_case(ops, kind, B, L, ldw, hop, lens=None, N=2048, win=2048, pad=None, sr=32000, n_mels=128, want=("spec", "mel", "cplx"),
             warp=True, seed=0, silent=()):
    """one forward launch against the float64 reference -> (x, float64 X, sum|a| per frame, frames per row, kernel outputs
    [spec, mel, cplx, ...]) for the adjoint"""
    pad = (N - hop) // 2 if pad is None else pad
    T, NB = n_frames(L, N, hop, pad), N // 2 + 1
    bk, fb = bank(ops, sr, N, n_mels)
    x, buf = wave(B, L, ldw, lens, seed, silent)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV) if lens is not None else None
    name = "mel_fwd_warp" if warp else "stft_fwd"
    tag = f"{name} N={N} win={win} pad={pad} hop={hop} B={B} L={L} ldw={ldw} mels={n_mels}"

    def run():
        spec, mel, cplx = run_fwd(ops, kind, buf, lens_d, B, L, ldw, N, hop, win, pad, T, bk, n_mels, want)
        outs = [body(spec, NB, tag + " spec") if spec is not None else None, body(mel, n_mels, tag + " mel") if mel is not None else None,
                cplx.cpu() if cplx is not None else None]
        if spec is not None and mel is not None:                       # spec_to_mel of the kernel's own |X|
            m2 = output(B * T, n_mels, n_mels + 1)
            ops._call("evk_spec_to_mel", P(spec), B * T, NB + 3, n_mels, P(bk.ptr), P(bk.idx), P(bk.val), P(m2), n_mels + 1)
            outs.append(body(m2, n_mels, tag + " spec_to_mel"))
        return [o for o in outs if o is not None], outs

    outs = run()[1]
    torch.cuda.synchronize()
    twice(lambda: run()[0])
    spec, mel, cplx = outs[0], outs[1], outs[2]
    X, A, counts = S.stft(x.double(), lens, N, hop, win, pad, T)
    past = torch.tensor([[f >= counts[b] for f in range(T)] for b in range(B)]).reshape(-1)
    ex = (past[:, None]).expand(-1, NB)

    def exact(e, m, val):
        return R.E(torch.where(m, torch.full_like(e.v, val), e.v), torch.where(m, torch.zeros_like(e.e), e.e))

    sp = S.spec_E(X, A, N, warp)
    sp = R.E(sp.v.reshape(B * T, NB), sp.e.reshape(B * T, NB))
    if spec is not None:
        chk(spec, exact(sp, ex, 0.0), tag + " |X|")
    if cplx is not None:
        eX = S.e_forward(A, N, warp).expand(B, T, NB).reshape(B * T, NB)
        ref = R.E(torch.view_as_real(X.reshape(B * T, NB)), torch.stack([eX, eX], -1))
        m2 = ex[..., None].expand(-1, -1, 2)
        chk(cplx, exact(ref, m2, 0.0), tag + " X")
    if mel is not None:
        lm = S.log_clip(S.mel_sum(sp, fb))
        chk(mel, exact(lm, past[:, None].expand(-1, n_mels), logf_clip()), tag + " log-mel")
        if spec is not None:
            assert torch.equal(outs[3].view(torch.int32), mel.view(torch.int32)), f"{tag}: spec_to_mel of |X| differs from the fused log-mel"
    return x, X, A, counts, outs


# ---- warp kernel: evk_mel_fwd at n_fft = win = 2048, pad = (2048 - hop) / 2 ------------------------------------------------------
# T = (L + 2 pad - 2048) / hop + 1.  The kernel is persistent: grid = min(ceil(B T / 6), 264) CTAs of 6 warps, so more than
# 264 * 6 = 1584 frames make a warp take a second frame (and prefetch it across the trip).
WARP_CASES = [
    # (B, L, ldw, hop, lens, sr, n_mels, want): the training segment, 8 x 32 frames
    (8, 20480, 20480, 640, None, 32000, 128, ("spec", "mel", "cplx")),
    # 4 x 500 = 2000 frames > 1584: second trips
    (4, 320000, 320000, 640, None, 32000, 128, ("mel",)),
    # row pitches 0, 1, 2, 3 mod 4: the cp.async (16 B), float2 (8 B) and scalar load paths
    (3, 20480, 20484, 640, None, 32000, 128, ("spec", "mel")),
    (3, 20480, 20485, 640, None, 32000, 128, ("spec", "mel")),
    (3, 20480, 20486, 640, None, 32000, 128, ("spec", "mel")),
    (3, 20480, 20487, 640, None, 32000, 128, ("spec", "mel")),
    # odd hops: pad 703 (641), 703 (642); frame starts alternate parity
    (2, 20000, 20003, 641, None, 32000, 128, ("spec", "mel", "cplx")),
    (2, 20000, 20002, 642, None, 32000, 128, ("spec", "mel")),
    # ragged: full, full - 1, a mid-frame end, a zero-frame row (< 640 = 2048 - 2 * 704), 0, the short row 650 (<= pad 704)
    (7, 12800, 12805, 640, [12800, 12799, 9000, 600, 0, 650, 11111], 32000, 128, ("spec", "mel", "cplx")),
    # B = 1 at an arbitrary length (a reference clip): (77777 + 1408 - 2048) / 640 + 1 = 121 frames
    (1, 77777, 77777, 640, None, 32000, 128, ("spec", "mel")),
    # other banks: 80 mels at 22.05 kHz (hop 256), 128 at 48 kHz (hop 480), 160 mels (> 143: the general-kernel fallback)
    (2, 30000, 30001, 256, None, 22050, 80, ("spec", "mel")),
    (2, 30000, 30002, 480, [30000, 17777], 48000, 128, ("spec", "mel")),
    (2, 20480, 20483, 640, [20480, 650], 32000, 160, ("spec", "mel", "cplx")),
    # one output at a time
    (2, 20480, 20480, 640, [20480, 10001], 32000, 128, ("spec",)),
    (2, 20480, 20480, 640, [20480, 10001], 32000, 128, ("cplx",)),
]


@pytest.mark.parametrize("case", range(len(WARP_CASES)))
def test_mel_fwd_warp(ops, case):
    B, L, ldw, hop, lens, sr, n_mels, want = WARP_CASES[case]
    fwd_case(ops, "mel", B, L, ldw, hop, lens, sr=sr, n_mels=n_mels, want=want, warp=n_mels <= 143, seed=case)


# ---- general kernel: evk_stft_fwd ---------------------------------------------------------------------------------------------------
# (N, win, pad, hop): every n_fft 256 .. 4096 (log2 N odd and even: 128 = 4^3 * 2 and 2048 = 4^5 * 2 packed points take the
# radix-2 pass), windows N, N / 2 and 256 centred, pads N / 2 (torch.stft center=True), (N - hop) / 2 and 0, hops 147, 160, 441, 640
GEN_CASES = [(256, 256, 128, 147), (256, 128, 48, 160), (256, 256, 0, 441), (512, 256, 0, 160), (512, 512, 256, 441),
             (1024, 512, 432, 160), (1024, 256, 0, 441), (1024, 1024, 512, 640), (2048, 1024, 1024, 147), (2048, 256, 704, 640),
             (4096, 4096, 2048, 441), (4096, 2048, 1728, 640), (4096, 256, 0, 147)]


@pytest.mark.parametrize("N,win,pad,hop", GEN_CASES, ids=[f"N{a}-win{b}-pad{c}-hop{d}" for a, b, c, d in GEN_CASES])
def test_stft_fwd_general(ops, N, win, pad, hop):
    L = 6 * N + 333
    # ragged: full, a mid-frame end, a row just past the padding, a row of pad samples (no frames), 0
    lens = [L, L - hop // 2 - 2 * N // 3, pad + N // 2 + 1, pad, 0]
    fwd_case(ops, "stft", 5, L, L + 3, hop, lens, N=N, win=win, pad=pad, sr=16000, n_mels=40 if N == 256 else 64, warp=False, seed=N + hop)


def test_mel_variant_general_at_training_geometry(ops):
    """evk_set_mel_variant(0): the training geometry on the general kernel, ragged, with the short row at b = 1"""
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_mel_variant(0)
    try:
        fwd_case(ops, "mel", 6, 20480, 20481, 640, [20480, 650, 20479, 9000, 600, 0], warp=False, seed=99)
    finally:
        lib.init().evk_set_mel_variant(1)


# ---- adjoint ----------------------------------------------------------------------------------------------------------------------
def bwd_check(ops, x, X, A, counts, lens, B, L, ldw, N, hop, win, pad, T, G, e_G, launch, tag, seed):
    base = torch.randn(B, L, generator=_gen(seed + 1))

    def run():
        dw = torch.full((B, ldw), SENTINEL)
        dw[:, :L] = base
        dw = dw.to(DEV)
        launch(dw)
        return [body(dw, L, tag + " dwav")]

    (got,) = twice(run)
    lens_eff = [L if lens is None else min(lens[b], L) for b in range(B)]
    fr, efr = S.inverse_frames(G, e_G, N, win)
    ref = S.ola(fr, efr, counts, lens_eff, L, N, hop, pad, base)
    chk(got, ref, tag + " dwav")
    return ref


def mel_bwd_case(ops, B, L, ldw, hop, lens, N=2048, win=2048, sr=32000, n_mels=128, silent=(), seed=0):
    pad = (N - hop) // 2
    T = n_frames(L, N, hop, pad)
    train = N == 2048 and win == 2048
    bk, fb = bank(ops, sr, N, n_mels)
    x, X, A, counts, outs = fwd_case(ops, "mel" if train else "stft", B, L, ldw, hop, lens, N=N, win=win, pad=pad, sr=sr, n_mels=n_mels,
                                     want=("mel", "cplx"), warp=train, seed=seed, silent=silent)
    mel, cplx = outs[1], outs[2]
    dmel = torch.randn(B * T, n_mels, generator=_gen(seed + 2))
    dmel_buf = torch.full((B * T, n_mels + 1), NAN)
    dmel_buf[:, :n_mels] = dmel
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV) if lens is not None else None
    mel_d = torch.full((B * T, n_mels + 2), NAN)
    mel_d[:, :n_mels] = mel
    dd, md, cd = dmel_buf.to(DEV), mel_d.to(DEV), cplx.to(DEV)

    def launch(dw):
        if train:
            ops._call("evk_mel_bwd", P(dd), n_mels + 1, P(cd), P(md), n_mels + 2, P(lens_d), B, L, ldw, hop, n_mels, P(bk.ptr), P(bk.idx),
                      P(bk.val), P(dw))
        else:
            ops._call("evk_stft_bwd", None, P(dd), n_mels + 1, P(cd), P(md), n_mels + 2, S.EPS, S.CLIP, n_mels, P(bk.ptr), P(bk.idx),
                      P(bk.val), P(lens_d), B, L, ldw, N, hop, win, pad, T, P(dw))

    G, e_G = S.mel_adjoint_G(X, A, N, fb, dmel.double().reshape(B, T, n_mels), warp=train)
    tag = f"{'mel_bwd' if train else 'stft_bwd'} N={N} win={win} hop={hop} lens={lens is not None}"
    ref = bwd_check(ops, x, X, A, counts, lens, B, L, ldw, N, hop, win, pad, T, G, e_G, launch, tag, seed)
    # the value of the model is the float64 autograd of the same expression
    xg = x.double().requires_grad_(True)
    Xg, _, _ = S.stft(xg, lens, N, hop, win, pad, T)
    (S.logmel_value(S.magnitude(Xg), fb) * dmel.double().reshape(B, T, n_mels)).sum().backward()
    lens_eff = [L if lens is None else min(lens[b], L) for b in range(B)]
    valid = torch.arange(L)[None, :] < torch.tensor(lens_eff)[:, None]
    assert torch.allclose(torch.where(valid, ref.v, torch.zeros_like(ref.v)),
                          torch.where(valid, xg.grad + torch.randn(B, L, generator=_gen(seed + 1)).double(), torch.zeros_like(ref.v)),
                          rtol=1e-9, atol=1e-9)


def test_mel_bwd_training(ops):
    """the training segment: 8 x 20480 (32 frames a row), row 3 silent: its dwav must come back as the base, bit for bit"""
    mel_bwd_case(ops, 8, 20480, 20481, 640, None, silent=(3,), seed=1)


def test_mel_bwd_training_ragged(ops):
    mel_bwd_case(ops, 6, 12800, 12803, 640, [12800, 650, 12799, 9000, 600, 0], silent=(2,), seed=2)


@pytest.mark.parametrize("ragged", [False, True])
def test_stft_bwd_logmel_1024(ops, ragged):
    """n_fft 1024, win 512, hop 160, 80 mels at 22.05 kHz: pad 432, (8000 + 864 - 1024) / 160 + 1 = 50 frames"""
    mel_bwd_case(ops, 4, 8000, 8002, 160, [8000, 7999, 4321, 433] if ragged else None, N=1024, win=512, sr=22050, n_mels=80, seed=3 + ragged)


# the MR-STFT loss: n_fft = max(win, 2048), hop 147, center=True (pad n_fft / 2); and 2048 / 441
CPLX_CASES = [(4096, 4096, 147), (2048, 2048, 147), (2048, 1024, 147), (2048, 512, 147), (2048, 256, 147), (2048, 2048, 441)]


@pytest.mark.parametrize("N,win,hop", CPLX_CASES, ids=[f"N{a}-win{b}-hop{c}" for a, b, c in CPLX_CASES])
def test_stft_bwd_complex(ops, N, win, hop):
    B, L, pad = 2, 9000, N // 2
    T, NB = n_frames(L, N, hop, pad), N // 2 + 1
    x, _ = wave(B, L, L + 1, None, N + win)
    X, A, counts = S.stft(x.double(), None, N, hop, win, pad, T)
    g = torch.randn(B * T, NB, 2, generator=_gen(win))
    gd = g.to(DEV)

    def launch(dw):
        ops._call("evk_stft_bwd", P(gd), None, 0, None, None, 0, 0.0, 0.0, 0, None, None, None, None, B, L, L + 1, N, hop, win, pad, T, P(dw))

    G = torch.view_as_complex(g.double().reshape(B, T, NB, 2).contiguous())
    ref = bwd_check(ops, x, X, A, counts, None, B, L, L + 1, N, hop, win, pad, T, G, torch.zeros(B, T, NB, dtype=torch.float64), launch,
                    f"stft_bwd N={N} win={win} hop={hop} cplx", win)
    xg = x.double().requires_grad_(True)
    Xg, _, _ = S.stft(xg, None, N, hop, win, pad, T)
    (Xg.real * G.real + Xg.imag * G.imag).sum().backward()
    base = torch.randn(B, L, generator=_gen(win + 1)).double()
    assert torch.allclose(ref.v, xg.grad + base, rtol=1e-9, atol=1e-9)


# ---- complex L1 -------------------------------------------------------------------------------------------------------------------
def test_cplx_l1(ops):
    """n = 132 * 8 * 256 + 12345 complex elements: 1056 blocks of 256 threads, a second grid-stride trip for the first 12345"""
    n = 132 * 8 * 256 + 12345
    g = _gen(11)
    a, b = torch.randn(n, 2, generator=g), torch.randn(n, 2, generator=g)
    b[::97] = a[::97]                                                  # a == b: gradient exactly 0
    base = float(torch.randn(1, generator=g))
    scale = 1.0 / n
    ad, bd = a.to(DEV), b.to(DEV)

    def run():
        loss = torch.tensor([base], device=DEV)
        grad = torch.full((n, 2), NAN, device=DEV)
        ops._call("evk_cplx_l1", P(ad), P(bd), n, scale, P(loss), P(grad))
        return [loss.cpu(), grad.cpu()]

    loss, grad = twice(run)
    rl, rg = S.cplx_l1(a, b, scale, base)
    chk(loss, R.E(rl.v.reshape(1), rl.e.reshape(1)), "cplx_l1 loss")
    chk(grad, rg, "cplx_l1 grad")


# ---- inverse STFT ------------------------------------------------------------------------------------------------------------------
ISTFT_CASES = [(2048, 441), (256, 64), (320, 80), (640, 160), (960, 240)]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("N,hop", ISTFT_CASES, ids=[f"N{a}-hop{b}" for a, b in ISTFT_CASES])
def test_istft_untrimmed(ops, N, hop, masked):
    """B = 2, S = 2, T = 12 frames: rows r = b S + s; the mask in the estimator's (b t (f s c)) layout, pitch 2 S NB + 2"""
    B, S_, T, NB = 2, 2, 12, N // 2 + 1
    g = _gen(N + masked)
    X = torch.randn(B * S_, T, NB, 2, generator=g)
    ldm = 2 * S_ * NB + 2
    mask = torch.full((B * T, ldm), NAN)
    mask[:, :2 * S_ * NB] = torch.randn(B * T, 2 * S_ * NB, generator=g)
    Lout = hop * (T - 1)
    Xd, md = X.to(DEV), mask.to(DEV)
    work = torch.empty(B * S_ * T * N, device=DEV)

    def run():
        out = output(B * S_, Lout, Lout + 3)
        ops._call("evk_istft", P(Xd), P(md) if masked else None, ldm if masked else 0, B, S_, T, N, hop, 0, P(work), P(out),
                  Lout + 3)
        return [body(out, Lout, "istft out")]

    (got,) = twice(run)
    Xc = torch.view_as_complex(X.double().contiguous())
    mc = None
    if masked:                                                         # row r = b S + s, frame t: mask[(b T + t), 2 (k S + s) + c]
        mm = mask[:, :2 * S_ * NB].double().reshape(B, T, NB, S_, 2).permute(0, 3, 1, 2, 4).reshape(B * S_, T, NB, 2)
        mc = torch.view_as_complex(mm.contiguous())
    ref, _ = S.istft(Xc, N, hop, mc)
    chk(got, ref, f"istft N={N} hop={hop} mask={masked}")
