"""GPU tests of Whisper transcription (`pytest -m gpu`): the log-mel kernel and the decode attention element for element against
float64, the encoder and teacher-forced decoder against the oracle (oracle/whisper_oracle.py) and the goldens that
oracle/pin_asr.py pinned against transformers, beam search end to end against `generate`'s tokens, batch invariance and
`WhisperAsr.recognize` on written wav files."""
import os

import numpy as np
import pytest
import torch

from oracle import pin_asr as PIN
from oracle import whisper_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "asr.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
# log-mel: fp32 DFT and mel sums against float64, in units of the normalised feature (1 = 4 decades of power).  Frames at
# the clamp (8 decades under the clip's max) carry the largest relative error of |X|^2.
TOL_MEL = 2e-3
# rel-L2 against float64, measured on an H100: encoder 5.3e-4 / 5.0e-4 with TF32 products, 1.2e-5 / 1.2e-5 under 3xTF32;
# teacher-forced logits 5.8e-4 / 7.2e-4 with TF32 products, 8.2e-6 / 9.3e-6 under 3xTF32
TOL_ENC, TOL_ENC_PRECISE = 5e-3, 5e-5
TOL_LOGITS, TOL_LOGITS_PRECISE = 5e-3, 5e-5


@pytest.fixture(scope="module")
def W():
    from easevoice_trainer_b200 import lib, whisper
    lib.init().evk_set_precise(0)
    return whisper


def precise(on):
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1 if on else 0)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def model(W, name):
    c = GOLD["cases"][name]
    net = W.WhisperModel(c["cfg"], GOLD["gen"])
    net.load_state_dict(PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"]))
    return net.to(DEV).eval(), c


def waves(c):
    return [PIN.clip(c["seed"] * 10 + i, s) for i, s in enumerate(c["secs"])]


def batch(xs):
    L = max(x.size for x in xs)
    w = torch.zeros(len(xs), L)
    for i, x in enumerate(xs):
        w[i, :x.size] = torch.from_numpy(x)
    return w.to(DEV), [x.size for x in xs]


@pytest.mark.parametrize("M", [80, 128])
def test_logmel_against_float64(W, M):
    fe = GOLD["frontend"][M]
    xs = [PIN.clip(fe["seed"], fe["secs"]), PIN.clip(7, 0.5), PIN.clip(8, 29.99)]
    net = W.WhisperModel(dict(W.LARGE_V3, num_mel_bins=M, d_model=128, encoder_attention_heads=2, decoder_attention_heads=2,
                              encoder_layers=1, decoder_layers=1, encoder_ffn_dim=128, decoder_ffn_dim=128,
                              vocab_size=PIN.vocab_size()), GOLD["gen"]).to(DEV)
    w, lens = batch(xs)
    got = net.features(w, lens).cpu()
    for i, x in enumerate(xs):
        ref = O.features(x, M)
        err = (got[i].double() - ref).abs().max().item()
        assert err <= TOL_MEL, (i, err)
        assert torch.all(got[i, O.num_frames(x.size):] == 0)


@pytest.mark.parametrize("name", ["m80_d2", "m128_d4"])
@pytest.mark.parametrize("prec", [False, True])
def test_encoder_and_decoder_against_oracle(W, name, prec):
    precise(prec)
    try:
        net, c = model(W, name)
        w, lens = batch(waves(c))
        feats = net.features(w, lens)
        ref_feats = torch.stack([O.features(x, c["cfg"]["num_mel_bins"]) for x in waves(c)])
        sd = PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"])
        enc_ref = O.encode(sd, ref_feats, c["cfg"])
        enc = net.encode(ref_feats.float().to(DEV))
        e = rel(enc, enc_ref)
        assert e <= (TOL_ENC_PRECISE if prec else TOL_ENC), e
        lg = net.teacher_forced_logits(enc, c["forced"].tolist())
        e2 = rel(lg, c["logits"])
        assert e2 <= (TOL_LOGITS_PRECISE if prec else TOL_LOGITS), e2
        print(f"{name} precise={prec}: encoder rel-L2 {e:.2e}, logits rel-L2 {e2:.2e}, feats max-abs "
              f"{(feats.cpu().double() - ref_feats).abs().max():.2e}")
    finally:
        precise(False)


def test_decode_attention_slot_tables(W):
    """Self-attention through slot tables, including a row that took another row's table (a beam reorder), and the
    cross-attention of a clip's beams, against float64."""
    from easevoice_trainer_b200 import ops
    g = torch.Generator().manual_seed(1)
    R, S, H, d = 6, 40, 3, 192
    pool = torch.randn(R * S, 2 * d, generator=g)
    tab = torch.randint(0, R * S, (R, S), generator=g, dtype=torch.int32)
    tab[3] = tab[1]                                   # row 3 reordered onto row 1's history
    q = torch.randn(R, 3 * d, generator=g)
    pos = 27
    out = ops.whisper_attn(q.to(DEV), pool.to(DEV), d, H, torch.empty(R, d, device=DEV), tab=tab.to(DEV),
                           pos=torch.tensor([pos], dtype=torch.int32, device=DEV), n_keys=S).cpu()
    for r in range(R):
        k = pool[tab[r, :pos + 1].long()].double()
        for h in range(H):
            qq = q[r, h * 64:(h + 1) * 64].double() * 0.125
            p = torch.softmax(k[:, h * 64:(h + 1) * 64] @ qq, 0)
            ref = p @ k[:, d + h * 64:d + (h + 1) * 64]
            assert (out[r, h * 64:(h + 1) * 64].double() - ref).abs().max() <= 1e-5
    # cross: 2 clips x 3 beams, 1500 keys
    ck = torch.randn(2 * 1500, 2 * d, generator=g)
    q2 = torch.randn(6, d, generator=g)
    o2 = ops.whisper_attn(q2.to(DEV), ck.to(DEV), d, H, torch.empty(6, d, device=DEV), n_keys=1500, nq=3).cpu()
    for r in range(6):
        k = ck[(r // 3) * 1500:(r // 3 + 1) * 1500].double()
        for h in range(H):
            p = torch.softmax(k[:, h * 64:(h + 1) * 64] @ (q2[r, h * 64:(h + 1) * 64].double() * 0.125), 0)
            assert (o2[r, h * 64:(h + 1) * 64].double() - p @ k[:, d + h * 64:d + (h + 1) * 64]).abs().max() <= 1e-5


def test_reordered_beam_equals_recomputed(W):
    """A beam that takes another parent mid-decode gives the logits of that hypothesis recomputed from scratch."""
    net, c = model(W, "m80_d2")
    precise(True)
    try:
        w, lens = batch(waves(c)[:1])
        enc = net.encode(net.features(w, lens))
        sp = net.sp
        a = [sp["sot"], sp["langs"]["en"], sp["transcribe"], sp["ts_begin"], 11, 12]
        b = [sp["sot"], sp["langs"]["en"], sp["transcribe"], sp["ts_begin"] + 2, 40, 41]
        st = net._state(1, 2, DEV)
        net.cross_kv(enc, st["ckv"])
        for t in range(5):
            st["pos"].fill_(t)
            st["tok"].copy_(torch.tensor([a[t], b[t]], dtype=torch.int32))
            net._forward_rows(st)
        # row 1 takes row 0's history (the table gather of the beam step), then both decode a[5]
        st["tab"][1] = st["tab"][0]
        st["pos"].fill_(5)
        st["tok"].fill_(a[5])
        lg = net._forward_rows(st).cpu()
        ref = net.teacher_forced_logits(enc, [a])[0, -1].cpu()
        assert torch.equal(lg[0], lg[1])
        assert rel(lg[1], ref) <= 1e-5          # 3xTF32 at 2 rows vs exact fp32 at 1 row: 1.3e-6 measured
    finally:
        precise(False)


@pytest.mark.parametrize("name", ["m80_d2", "m128_d4"])
def test_end_to_end_tokens_equal_generate(W, name):
    precise(True)
    try:
        net, c = model(W, name)
        feats = torch.stack([O.features(x, c["cfg"]["num_mel_bins"]) for x in waves(c)]).float().to(DEV)
        for run in c["runs"]:
            got = net.transcribe_features(feats, language=run["language"])
            for i, (o, r) in enumerate(zip(got, run["results"])):
                assert o["language"] == r["language"], (i, o["language"], r["language"])
                assert o["tokens"] == r["tokens"], (name, run["language"], i, o["tokens"], r["tokens"])
                assert abs(o["score"] - r["score"]) <= 1e-4 * max(1.0, abs(r["score"]))
                assert abs(o["no_speech_prob"] - r["no_speech_prob"]) <= 1e-4 * r["no_speech_prob"] + 1e-7
    finally:
        precise(False)


def test_batch_invariance(W):
    """A clip's encoder output and tokens are the same bits alone and in a batch of 8."""
    net, c = model(W, "m80_d2")
    xs = waves(c) + [PIN.clip(50 + i, 2.0 + 0.7 * i) for i in range(6)]
    w, lens = batch(xs)
    feats = net.features(w, lens)
    w1, l1 = batch(xs[:1])
    f1 = net.features(w1, l1)
    assert torch.equal(feats[:1], f1)
    enc8, enc1 = net.encode(feats), net.encode(f1)
    assert torch.equal(enc8[:1], enc1)
    t8 = net.transcribe_features(feats, language="en", enc=enc8)
    t1 = net.transcribe_features(f1, language="en", enc=enc1)
    assert t8[0] == t1[0]


def test_recognize_end_to_end(W, tmp_path):
    import json

    from scipy.io import wavfile

    from easevoice_trainer_b200 import asr
    c = GOLD["cases"]["m80_d2"]
    mdir = tmp_path / "model"
    mdir.mkdir()
    json.dump(dict(c["cfg"]), open(mdir / "config.json", "w"))
    json.dump(GOLD["gen"], open(mdir / "generation_config.json", "w"))
    torch.save(PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"]), mdir / "pytorch_model.bin")
    tok = asr_tokenizer(mdir, GOLD["n_text"])
    files = []
    for i, x in enumerate(waves(c)):
        f = str(tmp_path / f"clip{i}.wav")
        if i == 0:          # 32 kHz int16, as slicer.write_slices writes
            up = np.repeat(x, 2)
            wavfile.write(f, 32000, (np.clip(up, -1, 1) * 32767).astype(np.int16))
        else:
            wavfile.write(f, 16000, x.astype(np.float32))
        files.append(f)
    a = asr.WhisperAsr("large-v3", "zh", "float32", model_dir=str(mdir))
    out, dump = str(tmp_path / "asr.list"), str(tmp_path / "dump.list")
    res = a.recognize(files, out, dump)
    assert res.status == "success", res.message
    lines = open(out, encoding="utf-8").read().split("\n")
    assert len(lines) == 2 and all(ln.startswith(f + "|zh|") for ln, f in zip(lines, files))
    assert open(dump, encoding="utf-8").read() == open(out, encoding="utf-8").read()
    # the 16 kHz clip is the oracle's clip: its text is the decoded text tokens of generate's hypothesis
    want = [t for t in c["runs"][0]["results"][1]["tokens"] if t < GOLD["n_text"]]
    assert lines[1].split("|", 2)[2] == tok.decode(want)
    info = res.data[files[1]]
    assert set(info) >= {"status", "avg_logprob", "compression_ratio", "no_speech_prob"}


def asr_tokenizer(mdir, n_text):
    """A word-level tokenizer.json over the first n_text ids (word i is "w<i> "), written into mdir."""
    from tokenizers import Tokenizer, models
    vocab = {f"w{i}": i for i in range(n_text)}
    vocab["[UNK]"] = n_text
    t = Tokenizer(models.WordLevel(vocab=vocab, unk_token="[UNK]"))
    t.save(str(mdir / "tokenizer.json"))
    return Tokenizer.from_file(str(mdir / "tokenizer.json"))


def _beam_case(W, net, g, seed, max_length=3 + 224):
    """One evk_whisper_beam_step call on 4 clips x 5 beams of random logits against whisper_oracle.process + beam_step.
    Rows cover: no timestamp yet, a single timestamp after text (only timestamps or eot may follow), a timestamp pair, timestamp
    logits raised so that their mass wins (forced timestamp), eot raised (finished hypotheses); clip 3 already holds a full,
    good finished set, so the early-stop heuristic stops it.  -> (kernel state, oracle results, clips compared)."""
    from easevoice_trainer_b200 import ops
    sp, V, beam, clips, plen = net.sp, net.cfg["vocab_size"], 5, 4, 3
    tb, eot = sp["ts_begin"], sp["eot"]
    gen = torch.Generator().manual_seed(seed)
    R = clips * beam
    logits = 3 * torch.randn(R, V, generator=gen)
    logits[1::4, tb:] += 4.0                                  # timestamp mass wins
    logits[0::5, eot] += 12.0                                 # eot the best candidate of the best beam
    hists = []
    for r in range(R):
        h = [int(t) for t in torch.randint(0, GOLD["n_text"], (g,), generator=gen)]
        if g >= 2 and r % 3 == 1:
            h[-2], h[-1] = 17, tb + 5 + r                       # text then one timestamp
        elif g >= 2 and r % 3 == 2:
            h[-2], h[-1] = tb + 3, tb + 9                       # a timestamp pair
        hists.append(h)
    if g == 0:
        score = torch.tensor([0.0] + [O.NEG] * (beam - 1)).repeat(clips)
    else:
        # running scores best first, as _beam_search keeps them
        score = -(torch.rand(clips, beam, generator=gen) * 2 + 1).sort(dim=1)[0].reshape(-1) * g
    fin_sc = torch.full((clips, beam), O.NEG)
    fin_done = torch.zeros(clips, beam, dtype=torch.bool)
    fin_sq = [[[] for _ in range(beam)] for _ in range(clips)]
    if g > 0:
        fin_sc[3], fin_done[3] = -0.01, True
        fin_sq[3] = [[7, 8] for _ in range(beam)]
        fin_sc[1, 0], fin_done[1, 0], fin_sq[1][0] = -2.5, True, [9]
    st = net._state(clips, beam, DEV)
    S = st["S"]
    st["g"].fill_(g)
    st["pos"].fill_(plen - 1 + g)
    st["score"].copy_(score)
    hist = torch.zeros(R, S, dtype=torch.int32)
    for r, h in enumerate(hists):
        hist[r, :g] = torch.tensor(h, dtype=torch.int32)
    st["hist"].copy_(hist)
    tab = torch.randint(0, R * S, (R, S), generator=gen, dtype=torch.int32)
    st["tab"].copy_(tab)
    st["fin_score"].copy_(fin_sc)
    st["fin_flag"].copy_(fin_done.int())
    fs = torch.zeros(clips, beam, S, dtype=torch.int32)
    fl = torch.zeros(clips, beam, dtype=torch.int32)
    for c in range(clips):
        for j in range(beam):
            fs[c, j, :len(fin_sq[c][j])] = torch.tensor(fin_sq[c][j], dtype=torch.int32)
            fl[c, j] = len(fin_sq[c][j])
    st["fin_seq"].copy_(fs)
    st["fin_len"].copy_(fl)
    st["unsat"].fill_(1)
    mit = sp["max_initial_ts"]
    ops.whisper_beam_step(logits.to(DEV), st, beam, (eot, sp["notimestamps"], tb, -1 if mit is None else int(mit), plen, max_length))
    prompt = [sp["sot"], sp["langs"]["en"], sp["transcribe"]]
    lp_all = O.process(torch.log_softmax(logits, -1), hists, sp)
    refs, compared = [], []
    for c in range(clips):
        rows = slice(c * beam, (c + 1) * beam)
        lp = lp_all[rows]
        o = O.beam_step(lp, [prompt + hists[r] for r in range(c * beam, (c + 1) * beam)], score[rows].float(),
                        [prompt + s for s in fin_sq[c]], fin_sc[c].float(), fin_done[c].tolist(), True, plen, max_length, eot)
        o["lp"] = lp
        acc = (lp + score[rows, None]).reshape(-1)
        top = torch.topk(acc, 2 * beam + 1)[0]
        gaps = (top[:-1] - top[1:]).abs()
        # selections are compared where the margins exceed the fp32 difference of the two log_softmax implementations
        if bool((gaps[torch.isfinite(gaps)] > 1e-4).all()):
            compared.append(c)
        refs.append(o)
    return st, refs, compared, tab, lp_all


@pytest.mark.parametrize("g,seed,max_length", [(0, 1, 227), (6, 2, 227), (9, 3, 227), (4, 4, 8)])
def test_beam_step_against_oracle(W, g, seed, max_length):
    net, _ = model(W, "m80_d2")
    st, refs, compared, tab, lp_all = _beam_case(W, net, g, seed, max_length)
    assert len(compared) >= 3, compared
    beam, plen, S = 5, 3, st["S"]
    tok, par, sc = st["tok"].cpu(), st["parent"].cpu(), st["score"].cpu()
    fsc, ffl, fln, fsq = st["fin_score"].cpu(), st["fin_flag"].cpu(), st["fin_len"].cpu(), st["fin_seq"].cpu()
    hist, tab_new, unsat = st["hist"].cpu(), st["tab"].cpu(), st["unsat"].cpu()
    pos = plen - 1 + g
    for c in compared:
        o, r0 = refs[c], c * beam
        assert int(unsat[c]) == int(o["unsat"]), (c, int(unsat[c]), o["unsat"])
        assert ffl[c].bool().tolist() == o["fin_done"]
        for j in range(beam):
            if o["fin_done"][j]:
                assert abs(float(fsc[c, j]) - float(o["fin_sc"][j])) <= 1e-4 * max(1.0, abs(float(o["fin_sc"][j])))
                assert fsq[c, j, :int(fln[c, j])].tolist() == o["fin"][j][plen:]
        if max_length == plen + g + 1:
            # every candidate hit the length limit: the running beams all sit at score - 1e9, where float32 rounding makes
            # them tie; transformers ends the search here, so only the finished set above is the result
            continue
        assert tok[r0:r0 + beam].tolist() == o["tok"], (c, tok[r0:r0 + beam].tolist(), o["tok"])
        assert (par[r0:r0 + beam] - r0).tolist() == o["parent"]
        assert torch.allclose(sc[r0:r0 + beam], o["run_sc"], rtol=1e-5, atol=1e-4)
        for b in range(beam):
            assert hist[r0 + b, :g + 1].tolist() == o["run"][b][plen:]
            assert torch.equal(tab_new[r0 + b, :pos + 1], tab[r0 + o["parent"][b], :pos + 1])
    # the rule paths this case was built to reach
    tb = net.sp["ts_begin"]
    if g == 0:
        assert all(bool(torch.isinf(lp_all[r, :tb]).all()) for r in range(lp_all.shape[0]))
        assert all(bool(torch.isinf(lp_all[r, tb + 51:]).all()) for r in range(lp_all.shape[0]))
    else:
        forced = [r for r in range(lp_all.shape[0]) if bool(torch.isinf(lp_all[r, :tb]).all())]
        assert forced, "no row with a forced timestamp"
        assert not refs[3]["unsat"], "the early-stop heuristic did not stop clip 3"
    if max_length == plen + g + 1:
        assert all(all(o["fin_done"]) for o in refs[:3])
    elif g > 0:
        assert any(any(d for d in o["fin_done"]) for o in refs[:3] if o is not refs[1])


def test_forced_no_speech_gives_empty_text(W, tmp_path):
    """A model whose first pass puts almost all mass on <|nospeech|> (and whose generation config suppresses it, so every
    generated token is improbable) writes an empty text through recognize."""
    import json

    from scipy.io import wavfile

    from easevoice_trainer_b200 import asr
    c = GOLD["cases"]["m80_d2"]
    sp = O.special_tokens(GOLD["gen"])
    sd = PIN.make_state_dict(c["cfg"], c["seed"], 1.0)
    d = c["cfg"]["d_model"]
    b0 = torch.full((d,), 0.3)
    sd["model.decoder.layer_norm.weight"] = torch.full((d,), 0.01)
    sd["model.decoder.layer_norm.bias"] = b0
    sd["model.decoder.embed_tokens.weight"][sp["nospeech"]] = 5.0 * b0 / b0.norm()
    gen = dict(GOLD["gen"], suppress_tokens=GOLD["gen"]["suppress_tokens"] + [sp["nospeech"]])
    mdir = tmp_path / "model"
    mdir.mkdir()
    json.dump(dict(c["cfg"]), open(mdir / "config.json", "w"))
    json.dump(gen, open(mdir / "generation_config.json", "w"))
    torch.save(sd, mdir / "pytorch_model.bin")
    asr_tokenizer(mdir, GOLD["n_text"])
    f = str(tmp_path / "clip.wav")
    wavfile.write(f, 16000, waves(c)[1].astype(np.float32))
    out = str(tmp_path / "asr.list")
    res = asr.WhisperAsr("large-v3", "zh", "float32", model_dir=str(mdir)).recognize([f], out, str(tmp_path / "dump"))
    assert res.status == "success", res.message
    info = res.data[f]
    assert info["no_speech_prob"] > 0.6 and info["avg_logprob"] < -1.0, info
    assert open(out, encoding="utf-8").read() == f"{f}|zh|"
