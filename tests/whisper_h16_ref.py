"""Float64 restatement of Whisper with 16-bit Linears, as whisper.py runs them under a float16 / bfloat16 compute type: both
operands of every Linear -- the encoder's, the decoder's and the tied head -- rounded to nearest even to 16 bits, then
multiplied and summed in float64.  The activation is rounded from its fp32 value (the kernels stage fp32 activations), the
weight from the fp32 checkpoint.  Everything else is oracle/whisper_oracle.py's float64 computation."""
import torch

from oracle import whisper_oracle as O


def h16(x, dtype):
    """x rounded to fp32, then to nearest even in `dtype` (torch.float16 / torch.bfloat16), returned as float64."""
    return x.float().to(dtype).double()


def _lin(x, sd, p, dtype, bias=True):
    y = h16(x, dtype) @ h16(sd[p + ".weight"], dtype).T
    return y + sd[p + ".bias"] if bias else y


def _mha(x, kv, sd, p, H, causal, dtype):
    B, T, D = x.shape
    q = _lin(x, sd, p + ".q_proj", dtype).view(B, T, H, -1).transpose(1, 2)
    k = _lin(kv, sd, p + ".k_proj", dtype, bias=False).view(B, kv.shape[1], H, -1).transpose(1, 2)
    v = _lin(kv, sd, p + ".v_proj", dtype).view(B, kv.shape[1], H, -1).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * (D // H) ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool).triu(1), float("-inf"))
    a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, T, D)
    return _lin(a, sd, p + ".out_proj", dtype)


def encode(sd, feats, cfg, dtype):
    """whisper_oracle.encode with 16-bit Linears."""
    sd = {k: v.double() for k, v in sd.items()}
    x = feats.double().transpose(1, 2)
    x = O._gelu(torch.nn.functional.conv1d(x, sd["model.encoder.conv1.weight"], sd["model.encoder.conv1.bias"], padding=1))
    x = O._gelu(torch.nn.functional.conv1d(x, sd["model.encoder.conv2.weight"], sd["model.encoder.conv2.bias"], stride=2, padding=1))
    h = x.transpose(1, 2) + sd["model.encoder.embed_positions.weight"]
    H = cfg["encoder_attention_heads"]
    for i in range(cfg["encoder_layers"]):
        p = f"model.encoder.layers.{i}."
        a = O._ln(h, sd, p + "self_attn_layer_norm")
        h = h + _mha(a, a, sd, p + "self_attn", H, False, dtype)
        h = h + _lin(O._gelu(_lin(O._ln(h, sd, p + "final_layer_norm"), sd, p + "fc1", dtype)), sd, p + "fc2", dtype)
    return O._ln(h, sd, "model.encoder.layer_norm")


def decode_logits(sd, enc, tokens, cfg, dtype):
    """whisper_oracle.decode_logits with 16-bit Linears and head."""
    sd = {k: v.double() for k, v in sd.items()}
    T = tokens.shape[1]
    h = sd["model.decoder.embed_tokens.weight"][tokens] + sd["model.decoder.embed_positions.weight"][:T]
    H = cfg["decoder_attention_heads"]
    enc = enc.double()
    for i in range(cfg["decoder_layers"]):
        p = f"model.decoder.layers.{i}."
        a = O._ln(h, sd, p + "self_attn_layer_norm")
        h = h + _mha(a, a, sd, p + "self_attn", H, True, dtype)
        h = h + _mha(O._ln(h, sd, p + "encoder_attn_layer_norm"), enc, sd, p + "encoder_attn", H, False, dtype)
        h = h + _lin(O._gelu(_lin(O._ln(h, sd, p + "final_layer_norm"), sd, p + "fc1", dtype)), sd, p + "fc2", dtype)
    h = O._ln(h, sd, "model.decoder.layer_norm")
    return h16(h, dtype) @ h16(sd["model.decoder.embed_tokens.weight"], dtype).T


def transcribe_clip(sd, cfg, sp, feats, dtype, language=None, num_beams=5, max_new_tokens=224):
    """whisper_oracle.transcribe_clip with 16-bit Linears."""
    enc = encode(sd, feats[None], cfg, dtype)
    l0 = decode_logits(sd, enc, torch.tensor([[sp["sot"]]]), cfg, dtype)[0, -1]
    langs = sp["langs"]
    lang_ids = torch.tensor(sorted(langs.values()))
    if language is None:
        lid = int(lang_ids[l0[lang_ids].argmax()])
        language = {v: k for k, v in langs.items()}[lid]
    nsp = float(torch.softmax(l0, -1)[sp["nospeech"]])
    prompt = [sp["sot"], langs[language], sp["transcribe"]]

    def fn(rows):
        return decode_logits(sd, enc.expand(len(rows), -1, -1), torch.tensor(rows), cfg, dtype)[:, -1]

    toks, score = O.beam_search(fn, prompt, sp, num_beams, max_new_tokens)
    return dict(language=language, tokens=toks, score=score, no_speech_prob=nsp)
