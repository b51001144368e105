"""CPU tests of Whisper's 16-bit compute types: `WhisperAsr`'s precision mapping, the packed-weight cache key following the
compute type, and the float64 emulation of 16-bit Linears (tests/whisper_h16_ref.py) against a direct computation, with
round-to-nearest-even (not truncation) at exact fp16 and bf16 midpoints."""
import numpy as np
import pytest
import torch

from tests import whisper_h16_ref as R

SMALL = dict(num_mel_bins=80, d_model=128, encoder_layers=1, decoder_layers=1, encoder_attention_heads=2,
             decoder_attention_heads=2, encoder_ffn_dim=128, decoder_ffn_dim=128, vocab_size=1613, max_source_positions=1500,
             max_target_positions=448)


def test_precision_mapping(monkeypatch):
    from easevoice_trainer_b200 import asr, whisper
    assert asr.compute_dtype("float16") is torch.float16 and asr.compute_dtype("bfloat16") is torch.bfloat16
    for p in ("float32", "int8", "int8_float16", "int8_float32", "int8_bfloat16", "int16", "default", "auto"):
        assert asr.compute_dtype(p) is None, p
    seen = []

    def fake(path, device="cuda", compute_type=None):
        seen.append(compute_type)
        return object()
    monkeypatch.setattr(whisper.WhisperModel, "from_pretrained", staticmethod(fake))
    import tokenizers
    monkeypatch.setattr(tokenizers.Tokenizer, "from_file", staticmethod(lambda p: object()))
    for p in ("float16", "bfloat16", "float32", "int8_float16"):
        asr.WhisperAsr("large-v3", "en", p, model_dir="/nonexistent").load()
    assert seen == [torch.float16, torch.bfloat16, None, None]


def test_cache_key_follows_compute_type():
    from easevoice_trainer_b200 import whisper
    from oracle import pin_asr as PIN
    net = whisper.WhisperModel(SMALL, PIN.generation_config())
    k0 = net.weights_key()
    built = []
    net.cached("probe", lambda: built.append(1))
    net.cached("probe", lambda: built.append(1))
    assert len(built) == 1
    for dt in (torch.float16, torch.bfloat16):
        net.set_compute_type(dt)
        assert net.weights_key() != k0
        net.cached("probe", lambda: built.append(1))
    assert len(built) == 3
    net.set_compute_type(None)
    assert net.weights_key() == k0
    for bad in (torch.float32, "float16", torch.int8):
        with pytest.raises(ValueError):
            net.set_compute_type(bad)


def rne_bf16(a):
    """fp32 -> bf16 by round to nearest even on the bit pattern, as float64."""
    b = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).astype(np.float64)


def direct_h16(a, dtype):
    a = np.asarray(a, dtype=np.float32)
    return a.astype(np.float16).astype(np.float64) if dtype is torch.float16 else rne_bf16(a)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_emulation_against_direct_float64(dtype):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(7, 40, generator=g, dtype=torch.float64) * 3
    sd = {"l.weight": torch.randn(24, 40, generator=g, dtype=torch.float64), "l.bias": torch.randn(24, generator=g, dtype=torch.float64)}
    hx, hw = direct_h16(x.numpy(), dtype), direct_h16(sd["l.weight"].numpy(), dtype)
    assert np.array_equal(R.h16(x, dtype).numpy(), hx)
    want = hx @ hw.T + sd["l.bias"].numpy()
    got = R._lin(x, sd, "l", dtype).numpy()
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    # the rounding is real: the emulation is not the float64 product
    assert np.abs(got - (x.numpy() @ sd["l.weight"].numpy().T + sd["l.bias"].numpy())).max() > 1e-4


@pytest.mark.parametrize("dtype,ulp", [(torch.float16, 2.0 ** -10), (torch.bfloat16, 2.0 ** -7)])
def test_round_to_nearest_even_at_midpoints(dtype, ulp):
    """1 + ulp/2 lies halfway between 1 (even) and 1 + ulp (odd): RNE gives 1.  1 + 3 ulp/2 lies between 1 + ulp (odd) and
    1 + 2 ulp (even): RNE gives 1 + 2 ulp where truncation gives 1 + ulp.  The emulation and the weight pack both do RNE."""
    from easevoice_trainer_b200 import ops
    x = torch.tensor([1 + ulp / 2, 1 + 3 * ulp / 2, -(1 + 3 * ulp / 2), 1 + 3 * ulp / 2 + ulp / 64], dtype=torch.float32)
    want = torch.tensor([1.0, 1 + 2 * ulp, -(1 + 2 * ulp), 1 + 2 * ulp], dtype=torch.float64)
    assert torch.equal(R.h16(x, dtype), want)
    assert np.array_equal(direct_h16(x.numpy(), dtype), want.numpy())
    pw = ops.pack_weight_h16(x[None].repeat(3, 1), dtype)
    assert pw.w.dtype == dtype and pw.w.shape == (3, 64) and pw.K == 4
    assert torch.equal(pw.w[:, :4].double(), want[None].repeat(3, 1)) and torch.all(pw.w[:, 4:] == 0)
