"""Whisper transcription on the library's kernels: transformers' `WhisperForConditionalGeneration` (inference only) and the beam
search of its `generate(num_beams=5, return_timestamps=True, task="transcribe", max_new_tokens=224)`: short-form for clips of
at most 30 s, long-form (`transcribe_long`: 30 s windows moved by the predicted timestamps) for longer ones.

  front end   evk_whisper_logmel: 400-point periodic-Hann STFT (hop 160, centre reflect padding) as a direct DFT, |X|^2, the
              Slaney mel bank (fmax 8 kHz), log10, max(x, clip max - 8), (x + 4) / 4 over the clip's own frames; the
              [B, 3000, n_mels] buffer is zero after them (openai-whisper's pad_or_trim of the normalised log-mel)
  encoder     conv(k3) + GELU, conv(k3, stride 2) + GELU on the conv routes, channels-last; + sinusoidal positions; pre-LN
              layers on one packed QKV Linear (k has no bias) and evk_attn_pad_fwd with every length 1500; final LayerNorm
  cross K/V   one Linear over all decoder layers, once per clip; the beams of a clip read it (row r reads clip r / beam)
  decoder     one step of all rows: token + learned position, per layer causal self-attention on slot tables
              (evk_whisper_self_kv / evk_whisper_attn), cross-attention, MLP; final LayerNorm; logits from the tied token
              embedding; evk_whisper_beam_step.  The step is captured as a CUDA graph per batch shape and replayed.
  long-form   evk_whisper_logmel over the whole clip, clamped at the whole clip's max - 8; evk_whisper_window cuts the
              3000-frame window at each clip's seek; the windows of several clips are encoded and decoded together as above
              (evk_whisper_beam_step with its log-sum-exp buffers, which also yield transformers' avg_logprob), and each
              clip's seek moves on the host by transformers' _retrieve_segment rules.

Compute is fp32 storage with TF32 tensor-core products in the Linears and the encoder's attention (3xTF32 under
`evk_set_precise(1)`); the decode attention and the beam step are exact fp32.  With a 16-bit compute type
(`set_compute_type(torch.float16 / torch.bfloat16)`, faster-whisper's compute_type "float16" / "bfloat16") every Linear
-- encoder, cross K/V, decode step and head -- runs on the 16-bit kernels instead: weights packed once in 16 bits, activations
rounded to 16 bits as they are staged, fp32 accumulation and epilogue (evk_linear_h16 for the encoder and the cross K/V
projection, evk_linear_rows_h16 for the decode step).  Activations, LayerNorm, both attentions, the cross K/V buffer, the
convs and the beam step stay fp32 as above.  Special-token ids come from the generation config.  No CPU fallback.
"""
import json
import os

import numpy as np
import torch

from . import ops
from .models import ParamTree
from .weights import check_state_dict

N_FFT, HOP, N_FRAMES, N_CTX = 400, 160, 3000, 1500
MAX_SAMPLES = 30 * 16000
NUM_BEAMS, MAX_NEW_TOKENS = 5, 224
# transformers' long-form skip rule (generate(no_speech_threshold=0.6, logprob_threshold=-1.0)): a window whose first pass
# puts more than 0.6 on <|nospeech|> and whose best hypothesis averages below -1.0 log-prob per token adds no text
NO_SPEECH_THRESHOLD, LOGPROB_THRESHOLD = 0.6, -1.0
CONFIG_KEYS = ("num_mel_bins", "d_model", "encoder_layers", "decoder_layers", "encoder_attention_heads",
               "decoder_attention_heads", "encoder_ffn_dim", "decoder_ffn_dim", "vocab_size", "max_source_positions",
               "max_target_positions")
LARGE_V3 = dict(num_mel_bins=128, d_model=1280, encoder_layers=32, decoder_layers=32, encoder_attention_heads=20,
                decoder_attention_heads=20, encoder_ffn_dim=5120, decoder_ffn_dim=5120, vocab_size=51866,
                max_source_positions=1500, max_target_positions=448)


def mel_filters(n_mels):
    """Slaney mel bank [201, n_mels] (transformers' mel_filter_bank(201, n_mels, 0, 8000, 16000, "slaney", "slaney"))."""
    def hz2mel(f):
        return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-12) / 1000.0) * (27.0 / np.log(6.4)), 3.0 * f / 200.0)

    def mel2hz(m):
        return np.where(m >= 15.0, 1000.0 * np.exp(np.log(6.4) / 27.0 * (m - 15.0)), 200.0 * m / 3.0)

    ff = mel2hz(np.linspace(hz2mel(np.float64(0.0)), hz2mel(np.float64(8000.0)), n_mels + 2))
    fft = np.linspace(0, 8000, N_FFT // 2 + 1)
    slopes = ff[None, :] - fft[:, None]
    d = np.diff(ff)
    fb = np.maximum(0.0, np.minimum(-slopes[:, :-2] / d[:-1], slopes[:, 2:] / d[1:]))
    return fb * (2.0 / (ff[2:] - ff[:-2]))[None, :]


def dft_basis():
    """[2, 400, 201]: periodic Hann * cos and -Hann * sin of the 400-point DFT, computed in float64."""
    n = np.arange(N_FFT)[:, None]
    k = np.arange(N_FFT // 2 + 1)[None, :]
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N_FFT) / N_FFT)
    ang = 2 * np.pi * ((n * k) % N_FFT) / N_FFT
    return np.stack([win[:, None] * np.cos(ang), -win[:, None] * np.sin(ang)])


def special_tokens(gen):
    """Special-token ids from a generation_config.json mapping (never constants)."""
    nots = int(gen["no_timestamps_token_id"])
    langs = {k[2:-2]: int(v) for k, v in gen["lang_to_id"].items()}
    return dict(sot=int(gen["decoder_start_token_id"]), eot=int(gen["eos_token_id"]), notimestamps=nots, ts_begin=nots + 1,
                nospeech=nots - 1, transcribe=int(gen["task_to_id"]["transcribe"]), langs=langs,
                suppress=[int(t) for t in gen.get("suppress_tokens") or []],
                begin_suppress=[int(t) for t in gen.get("begin_suppress_tokens") or []],
                max_initial_ts=gen.get("max_initial_timestamp_index"))


def retrieve_segment(seq, ts_begin, n_frames):
    """transformers' WhisperGenerationMixin._retrieve_segment for one window's best hypothesis seq (generated ids without the
    eot it ended on) -> (the tokens kept: those of its segments, how many frames seek moves).  A hypothesis with a pair of
    consecutive timestamps that does not end in a single timestamp keeps the tokens up to its last pair and moves seek to the
    pair's first timestamp (2 frames per 20 ms step); otherwise it keeps every token and seek moves by the whole window."""
    ts = [t >= ts_begin for t in seq]
    single_ending = ts[-2:] == [False, True]
    pairs = [i + 1 for i in range(len(seq) - 1) if ts[i] and ts[i + 1]]
    if not pairs or single_ending:
        return list(seq), n_frames
    last = pairs[-1] + 1
    return list(seq[:last]), (seq[last - 2] - ts_begin) * 2


class WhisperModel(ParamTree):
    """WhisperForConditionalGeneration (modeling_whisper.py) for inference, any size: shapes from the config, special tokens
    from the generation config."""

    def __init__(self, config, generation_config):
        super().__init__()
        c = dict(config)
        missing = [k for k in CONFIG_KEYS if k not in c]
        if missing:
            raise ValueError(f"config lacks {missing}")
        c = {k: int(c[k]) for k in CONFIG_KEYS}
        for side in ("encoder", "decoder"):
            if c["d_model"] != 64 * c[f"{side}_attention_heads"]:
                raise ValueError(f"{side}: head dim {c['d_model'] / c[f'{side}_attention_heads']} (the kernels take 64)")
        if c["max_source_positions"] != N_CTX or c["num_mel_bins"] % 4:
            raise ValueError("max_source_positions must be 1500 and num_mel_bins a multiple of 4")
        self.cfg, self.gen, self.sp = c, dict(generation_config), special_tokens(generation_config)
        self.compute_type = None
        if not (self.sp["ts_begin"] + 1501 <= c["vocab_size"] and self.sp["eot"] < self.sp["ts_begin"]):
            raise ValueError("generation config's token layout does not fit the vocabulary")
        for name, shape in self.param_spec(c):
            self._register(name, torch.ones(shape) if name.endswith("layer_norm.weight") else torch.zeros(shape))

    @staticmethod
    def param_spec(c):
        """(name, shape) of WhisperForConditionalGeneration's state_dict, without the tied proj_out.weight."""
        d, M, V = c["d_model"], c["num_mel_bins"], c["vocab_size"]
        out = [("model.encoder.conv1.weight", (d, M, 3)), ("model.encoder.conv1.bias", (d,)),
               ("model.encoder.conv2.weight", (d, d, 3)), ("model.encoder.conv2.bias", (d,)),
               ("model.encoder.embed_positions.weight", (c["max_source_positions"], d))]

        def attn(p):
            r = []
            for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
                r.append((p + n + ".weight", (d, d)))
                if n != "k_proj":
                    r.append((p + n + ".bias", (d,)))
            return r

        def block(p, ffn, cross):
            r = attn(p + "self_attn.") + [(p + "self_attn_layer_norm.weight", (d,)), (p + "self_attn_layer_norm.bias", (d,))]
            if cross:
                r += attn(p + "encoder_attn.") + [(p + "encoder_attn_layer_norm.weight", (d,)),
                                                  (p + "encoder_attn_layer_norm.bias", (d,))]
            return r + [(p + "fc1.weight", (ffn, d)), (p + "fc1.bias", (ffn,)), (p + "fc2.weight", (d, ffn)),
                        (p + "fc2.bias", (d,)), (p + "final_layer_norm.weight", (d,)), (p + "final_layer_norm.bias", (d,))]

        for i in range(c["encoder_layers"]):
            out += block(f"model.encoder.layers.{i}.", c["encoder_ffn_dim"], False)
        out += [("model.encoder.layer_norm.weight", (d,)), ("model.encoder.layer_norm.bias", (d,)),
                ("model.decoder.embed_tokens.weight", (V, d)),
                ("model.decoder.embed_positions.weight", (c["max_target_positions"], d))]
        for i in range(c["decoder_layers"]):
            out += block(f"model.decoder.layers.{i}.", c["decoder_ffn_dim"], True)
        return out + [("model.decoder.layer_norm.weight", (d,)), ("model.decoder.layer_norm.bias", (d,))]

    # ---- loading ----------------------------------------------------------------------------------------------------------
    def load_state_dict(self, sd, strict=True):
        """Strict: a missing or unexpected key, a non-float tensor or a wrong shape raises ValueError.  proj_out.weight, when
        present, must equal the token embedding it is tied to."""
        sd = dict(sd)
        tied = sd.pop("proj_out.weight", None)
        check_state_dict(sd, dict(self.param_spec(self.cfg)), "WhisperModel")
        if tied is not None and not torch.equal(tied.float(), sd["model.decoder.embed_tokens.weight"].float()):
            raise ValueError("proj_out.weight differs from model.decoder.embed_tokens.weight (untied heads are not supported)")
        return super().load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)

    def set_compute_type(self, dtype):
        """None: fp32 storage with TF32 products (the default); torch.float16 or torch.bfloat16: every Linear on the 16-bit
        kernels.  The packed weights and the captured step graphs follow on the next call.  -> self."""
        if dtype is not None and dtype not in ops.H16_TYPES:
            raise ValueError(f"compute type {dtype!r} (None, torch.float16 or torch.bfloat16)")
        self.compute_type = dtype
        return self

    def weights_key(self):
        """ParamTree's key and the compute type: a switch repacks the weights and captures the step graphs again."""
        return super().weights_key() + (str(self.compute_type),)

    @classmethod
    def from_pretrained(cls, path, device="cuda", compute_type=None):
        """A local Hugging Face directory: config.json, model.safetensors or pytorch_model.bin, generation_config.json.
        compute_type: as set_compute_type."""
        for f in ("config.json", "generation_config.json"):
            if not os.path.exists(os.path.join(path, f)):
                raise FileNotFoundError(os.path.join(path, f))
        net = cls(json.load(open(os.path.join(path, "config.json"))), json.load(open(os.path.join(path, "generation_config.json"))))
        st, pt = os.path.join(path, "model.safetensors"), os.path.join(path, "pytorch_model.bin")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        elif os.path.exists(pt):
            sd = torch.load(pt, map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin under {path}")
        net.load_state_dict(sd)
        return net.set_compute_type(compute_type).to(device).eval()

    # ---- packed operands --------------------------------------------------------------------------------------------------
    def _packed(self):
        """Every packed weight, made once per weights_key()."""
        return self.cached("packed", self._pack)

    def _pack(self):
        cfg, P, h16 = self.cfg, self.P, self.compute_type
        pk32 = lambda w: ops.pack_weight(w.detach().contiguous(), None, need_pb=False)   # noqa: E731
        # the Linears' operand: the fp32 (TF32) pack, or only the 16-bit one
        pk = pk32 if h16 is None else lambda w: ops.pack_weight_h16(w, h16)           # noqa: E731
        z = lambda n: torch.zeros(n, device=P("model.encoder.conv1.bias").device)     # noqa: E731
        d = {}

        def lin(name, pack=pk):
            d[name] = (pack(P(name + ".weight")), P(name + ".bias").detach())

        def qkv(p):
            w = torch.cat([P(p + n + ".weight") for n in ("q_proj", "k_proj", "v_proj")])
            d[p + "qkv"] = (pk(w), torch.cat([P(p + "q_proj.bias"), z(cfg["d_model"]), P(p + "v_proj.bias")]).detach())

        lin("model.encoder.conv1", pk32)
        lin("model.encoder.conv2", pk32)
        for i in range(cfg["encoder_layers"]):
            p = f"model.encoder.layers.{i}."
            qkv(p + "self_attn.")
            for n in ("self_attn.out_proj", "fc1", "fc2"):
                lin(p + n)
        ws, bs = [], []
        for i in range(cfg["decoder_layers"]):
            p = f"model.decoder.layers.{i}."
            qkv(p + "self_attn.")
            for n in ("self_attn.out_proj", "encoder_attn.q_proj", "encoder_attn.out_proj", "fc1", "fc2"):
                lin(p + n)
            ws += [P(p + "encoder_attn.k_proj.weight"), P(p + "encoder_attn.v_proj.weight")]
            bs += [z(cfg["d_model"]), P(p + "encoder_attn.v_proj.bias")]
        d["cross_kv"] = (pk(torch.cat(ws)), torch.cat(bs).detach())
        d["head"] = pk(P("model.decoder.embed_tokens.weight"))
        dev = P("model.encoder.conv1.bias").device
        d["basis"] = torch.tensor(dft_basis(), dtype=torch.float32, device=dev).contiguous()
        d["fb"] = torch.tensor(mel_filters(cfg["num_mel_bins"]), dtype=torch.float32, device=dev).contiguous()
        return d

    def _ln(self, x, name):
        return ops.whisper_layernorm(x, self.P(name + ".weight"), self.P(name + ".bias"), eps=1e-5)

    def _linear(self, x, wb, act=ops.ACT_NONE, res=None, rows=False):
        """One Linear of the packed (w, b) on the compute type's kernels: TF32 (ops.linear), or 16 bits with the row kernel for
        the decode step (rows=True) and the wgmma kernel otherwise."""
        w, b = wb
        if self.compute_type is None:
            return ops.linear(x, w, b, act=act, res=res)
        return (ops.linear_rows_h16 if rows else ops.linear_h16)(x, w, b, act=act, res=res)

    # ---- front end and encoder --------------------------------------------------------------------------------------------
    @torch.no_grad()
    def features(self, wav, lens):
        """wav [B, L] fp32 device 16 kHz (row b holds lens[b] samples, 201 <= lens[b] <= 480000) -> [B, 3000, n_mels]."""
        lens = [int(n) for n in lens]
        for b, n in enumerate(lens):
            if not (N_FFT // 2 + 1 <= n <= min(MAX_SAMPLES, wav.shape[1])):
                raise ValueError(f"row {b}: {n} samples (a clip takes 201 .. 480000 samples of 16 kHz audio)")
        pk = self._packed()
        ln = torch.tensor(lens, dtype=torch.int32).to(wav.device)
        return ops.whisper_logmel(wav.float().contiguous(), ln, N_FRAMES, pk["basis"], pk["fb"])

    @torch.no_grad()
    def features_long(self, wav, lens):
        """wav [B, L] fp32 device 16 kHz (row b holds lens[b] >= 201 samples, any length) -> [B, max lens // 160, n_mels]: the
        log-mel of each whole clip normalised with its own max over all its frames, zero after its lens[b] // 160 frames."""
        lens = [int(n) for n in lens]
        for b, n in enumerate(lens):
            if not (N_FFT // 2 + 1 <= n <= wav.shape[1]):
                raise ValueError(f"row {b}: {n} samples (a clip takes at least 201 samples of 16 kHz audio)")
        pk = self._packed()
        ln = torch.tensor(lens, dtype=torch.int32).to(wav.device)
        return ops.whisper_logmel(wav.float().contiguous(), ln, max(lens) // HOP, pk["basis"], pk["fb"])

    @torch.no_grad()
    def encode(self, feats):
        """feats [B, 3000, n_mels] -> encoder last_hidden_state [B, 1500, d_model]."""
        c, pk = self.cfg, self._packed()
        B = feats.shape[0]
        w, b = pk["model.encoder.conv1"]
        x = ops.gelu(ops.conv(feats.contiguous(), w, b, pad=1))
        w, b = pk["model.encoder.conv2"]
        # one launch per clip: the stride-2 conv takes evk_gconv_fwd's phase-split route from 2048 output rows on, so a
        # batched launch would round differently from a clip alone
        x = torch.cat([ops.gelu(ops.conv(x[i:i + 1], w, b, stride=2, pad=1)) for i in range(B)]).contiguous()
        ops.whisper_add_pos(x, self.P("model.encoder.embed_positions.weight").detach())
        lens = torch.full((B,), N_CTX, dtype=torch.int64, device=x.device)
        H = c["encoder_attention_heads"]
        for i in range(c["encoder_layers"]):
            p = f"model.encoder.layers.{i}."
            qkv = self._linear(self._ln(x, p + "self_attn_layer_norm"), pk[p + "self_attn.qkv"])
            a = ops.attention_pad(qkv, heads=H, lens=lens, scale=0.125)
            x = self._linear(a, pk[p + "self_attn.out_proj"], res=x)
            f = self._linear(self._ln(x, p + "final_layer_norm"), pk[p + "fc1"], act=ops.ACT_GELU)
            x = self._linear(f, pk[p + "fc2"], res=x)
        return self._ln(x, "model.encoder.layer_norm")

    @torch.no_grad()
    def cross_kv(self, enc, out):
        """Writes out [B * 1500, decoder_layers * 2 * d_model]: layer l's K at columns 2 d l, V at 2 d l + d."""
        w, b = self._packed()["cross_kv"]
        x = enc.reshape(-1, enc.shape[-1]).contiguous()
        if self.compute_type is None:
            return ops.linear_into(x, w, out, b)
        return ops.linear_h16(x, w, b, out=out)

    # ---- decoding ---------------------------------------------------------------------------------------------------------
    def _state(self, clips, beam, dev):
        c, sp = self.cfg, self.sp
        R, S, d, Ld = clips * beam, c["max_target_positions"], c["d_model"], c["decoder_layers"]
        it = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)     # noqa: E731
        return dict(clips=clips, beam=beam, R=R, S=S, pos=it(1), g=it(1), tok=it(R), parent=it(R), hist=it(R, S), tab=it(R, S),
                    x=torch.zeros(R, d, device=dev), pool=torch.zeros(R * S, Ld * 2 * d, device=dev),
                    ckv=torch.zeros(clips * N_CTX, Ld * 2 * d, device=dev), score=torch.zeros(R, device=dev),
                    cv=torch.zeros(R, 2 * beam, device=dev), ci=it(R, 2 * beam), fin_score=torch.zeros(clips, beam, device=dev),
                    fin_seq=it(clips, beam, S), fin_len=it(clips, beam), fin_flag=it(clips, beam), unsat=it(clips),
                    nsp=torch.zeros(R, device=dev), lang_tok=it(R), row_lse=torch.zeros(R, device=dev),
                    run_lse=torch.zeros(R, device=dev), fin_lse=torch.zeros(clips, beam, device=dev),
                    sup=torch.tensor(sp["suppress"], dtype=torch.int32, device=dev),
                    bsup=torch.tensor(sp["begin_suppress"], dtype=torch.int32, device=dev),
                    lang_ids=torch.tensor(sorted(sp["langs"].values()), dtype=torch.int32, device=dev))

    def _forward_rows(self, st):
        """Logits [R, V] of every row's token st["tok"] at position st["pos"], its K / V appended to its slot table."""
        c, pk = self.cfg, self._packed()
        R, S, d, H, beam = st["R"], st["S"], c["d_model"], c["decoder_attention_heads"], st["beam"]
        x = ops.whisper_embed(st["tok"], self.P("model.decoder.embed_tokens.weight").detach(),
                              self.P("model.decoder.embed_positions.weight").detach(), st["pos"], st["x"])
        for i in range(c["decoder_layers"]):
            p = f"model.decoder.layers.{i}."
            qkv = self._linear(self._ln(x, p + "self_attn_layer_norm"), pk[p + "self_attn.qkv"], rows=True)
            pool = st["pool"][:, 2 * d * i:]
            ops.whisper_self_kv(qkv, pool, st["tab"], st["pos"], S)
            a = ops.whisper_attn(qkv, pool, d, H, torch.empty(R, d, device=x.device), tab=st["tab"], pos=st["pos"], n_keys=S)
            x = self._linear(a, pk[p + "self_attn.out_proj"], res=x, rows=True)
            q = self._linear(self._ln(x, p + "encoder_attn_layer_norm"), pk[p + "encoder_attn.q_proj"], rows=True)
            a = ops.whisper_attn(q, st["ckv"][:, 2 * d * i:], d, H, torch.empty(R, d, device=x.device), n_keys=N_CTX, nq=beam)
            x = self._linear(a, pk[p + "encoder_attn.out_proj"], res=x, rows=True)
            f = self._linear(self._ln(x, p + "final_layer_norm"), pk[p + "fc1"], act=ops.ACT_GELU, rows=True)
            x = self._linear(f, pk[p + "fc2"], res=x, rows=True)
        return self._linear(self._ln(x, "model.decoder.layer_norm"), (pk["head"], None), rows=True)

    def _layout(self, plen, max_new_tokens):
        sp = self.sp
        mit = sp["max_initial_ts"]
        return (sp["eot"], sp["notimestamps"], sp["ts_begin"], -1 if mit is None else int(mit), plen, plen + max_new_tokens)

    def _graph(self, clips, beam, dev, max_new_tokens, track_lse=False):
        """The decode step (forward of every row, beam step, position + 1) captured once per (clips, beam, max_new_tokens,
        track_lse).  Graphs of one (clips, beam) share one decode state; a batch of another shape replaces that state and its
        graphs rather than adding to the device memory a batch is sized for (cross K/V and slots for every clip).  track_lse:
        the beam step also carries what transformers' long-form avg_logprob needs.  The graphs hold the packed operands and the
        precise mode's kernels, so they are captured again whenever _packed() is made again."""
        graphs = self.cached("graphs", dict)
        skey = (clips, beam, str(dev))
        if self.__dict__.get("_gstate") is None or self._gstate[0] != skey:
            graphs.clear()
            self._gstate = None
            torch.cuda.empty_cache()
            self._gstate = (skey, self._state(clips, beam, dev))
        gkey = (max_new_tokens, track_lse)
        if gkey in graphs:
            return graphs[gkey]
        st = self._gstate[1]
        lay = self._layout(3, max_new_tokens)

        def step():
            lg = self._forward_rows(st)
            ops.whisper_beam_step(lg, st, beam, lay, track_lse=track_lse)
            st["pos"].add_(1)
            st["g"].add_(1)
            return lg

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                # outside capture: allocator, lazy inits, shared-memory opt-ins
            step()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        graphs[gkey] = (g, st)
        return graphs[gkey]

    @torch.no_grad()
    def transcribe_features(self, feats, language=None, num_beams=NUM_BEAMS, max_new_tokens=MAX_NEW_TOKENS, check_every=8,
                            enc=None):
        """Beam search of a batch of clips.  feats [B, 3000, n_mels]; language: a code of the generation config's lang_to_id, a
        list of them (one per clip) or None (detected per clip by the argmax over the language tokens at
        <|startoftranscript|>).  -> list of dict(language, tokens (generated ids, eot included when the hypothesis ended on
        it), score (sum of log-probs / number of tokens: the length-normalised beam score), no_speech_prob)."""
        sp, c = self.sp, self.cfg
        B, dev = feats.shape[0], feats.device
        if max_new_tokens + 3 > c["max_target_positions"]:
            raise ValueError(f"max_new_tokens {max_new_tokens} + 3 prompt tokens exceed {c['max_target_positions']} positions")
        langs = [language] * B if language is None or isinstance(language, str) else list(language)
        for lg in langs:
            if lg is not None and lg not in sp["langs"]:
                raise ValueError(f"language {lg!r} is not in the generation config")
        enc = self.encode(feats) if enc is None else enc
        return self._decode(enc, langs, num_beams, max_new_tokens, check_every)[0]

    def _decode(self, enc, langs, num_beams, max_new_tokens, check_every, active=None, track_lse=False):
        """Beam search of the clips of enc [B, 1500, d] (langs: a code or None per clip).  active: 0 / 1 per clip; a clip with
        0 is finished before the first step, so it adds no steps and its result is empty.  track_lse: each result also has
        avg_logprob, transformers' long-form mean of log_softmax(processed row)[token] over the hypothesis' tokens.
        -> (results, number of decode steps)."""
        sp = self.sp
        B, dev = enc.shape[0], enc.device
        g, st = self._graph(B, num_beams, dev, max_new_tokens, track_lse)
        self.cross_kv(enc, st["ckv"])
        for k in ("hist", "tab", "fin_seq", "fin_len", "fin_flag", "pos", "g"):
            st[k].zero_()
        st["unsat"].fill_(1)
        if active is not None:
            st["unsat"].copy_(torch.tensor(active, dtype=torch.int32))
        if track_lse:
            st["run_lse"].zero_()
            st["fin_lse"].zero_()
        st["fin_score"].fill_(-1.0e9)
        st["score"].fill_(-1.0e9)
        st["score"].view(B, num_beams)[:, 0] = 0.0
        # prompt: <|startoftranscript|> (no-speech probability, language), the language, <|transcribe|>
        st["tok"].fill_(sp["sot"])
        ops.whisper_first_pass(self._forward_rows(st), sp["nospeech"], st["lang_ids"], st["nsp"], st["lang_tok"])
        forced = torch.tensor([sp["langs"][lg] if lg is not None else -1 for lg in langs], dtype=torch.int32, device=dev)
        forced = forced.repeat_interleave(num_beams)
        st["tok"].copy_(torch.where(forced >= 0, forced, st["lang_tok"]))
        lang_rows = st["tok"].view(B, num_beams)[:, 0].tolist()
        st["pos"].fill_(1)
        self._forward_rows(st)
        st["pos"].fill_(2)
        st["tok"].fill_(sp["transcribe"])
        steps = 0
        for n in range(max_new_tokens):
            g.replay()
            steps += 1
            if (n + 1) % check_every == 0 and not bool(st["unsat"].any()):
                break
        inv = {v: k for k, v in sp["langs"].items()}
        fin_len, fin_seq = st["fin_len"][:, 0].tolist(), st["fin_seq"][:, 0].tolist()
        sc, nsp = st["fin_score"][:, 0].tolist(), st["nsp"].view(B, num_beams)[:, 0].tolist()
        out = [dict(language=inv[lang_rows[b]], tokens=fin_seq[b][:fin_len[b]], score=sc[b], no_speech_prob=nsp[b])
               for b in range(B)]
        if track_lse:
            for o, lse in zip(out, st["fin_lse"][:, 0].tolist()):
                o["avg_logprob"] = o["score"] - lse / max(1, len(o["tokens"]))
        return out, steps

    @torch.no_grad()
    def transcribe_long(self, lm, frames, language=None, clips_per_batch=8, num_beams=NUM_BEAMS, max_new_tokens=MAX_NEW_TOKENS,
                        check_every=8):
        """Long-form transcription of a pool of clips: transformers' long-form `generate` (temperature 0 only, no conditioning
        on the previous window, no_speech_threshold 0.6, logprob_threshold -1.0) for each clip on its own.

        lm [P, T, n_mels]: features_long of the pool; frames[i]: clip i's frame count.  language: a code, a list of them or
        None (detected per clip on its first window, then forced on its later windows).  Each round takes the next window of
        up to clips_per_batch unfinished clips, round-robin over the pool, and decodes them as one batch of
        min(clips_per_batch, P) rows (one captured graph per pool); rows without a window are finished before the first step.
        -> per clip dict(language, tokens: the kept tokens of its windows in order, windows: per window dict(seek, n_frames,
        tokens (the best hypothesis), kept, score, avg_logprob, no_speech_prob, skipped, steps (decode steps of its round)))."""
        sp = self.sp
        P = len(frames)
        langs = [language] * P if language is None or isinstance(language, str) else list(language)
        for lg in langs:
            if lg is not None and lg not in sp["langs"]:
                raise ValueError(f"language {lg!r} is not in the generation config")
        if max_new_tokens + 3 > self.cfg["max_target_positions"]:
            raise ValueError(f"max_new_tokens {max_new_tokens} + 3 prompt tokens exceed {self.cfg['max_target_positions']} positions")
        frames = [int(f) for f in frames]
        nb, dev = max(1, min(int(clips_per_batch), P)), lm.device
        seek, windows, cursor = [0] * P, [[] for _ in range(P)], 0
        while True:
            pick = [i for i in ((cursor + k) % P for k in range(P)) if seek[i] < frames[i]][:nb]
            if not pick:
                break
            cursor = (pick[-1] + 1) % P
            n = [min(N_FRAMES, frames[i] - seek[i]) for i in pick]
            idle = nb - len(pick)
            tab = torch.tensor([[i, seek[i], k] for i, k in zip(pick, n)] + [[0, 0, 0]] * idle, dtype=torch.int32).to(dev)
            enc = self.encode(ops.whisper_window(lm, tab)[:len(pick)])
            if idle:
                enc = torch.cat([enc, enc.new_zeros((idle,) + tuple(enc.shape[1:]))])
            res, steps = self._decode(enc, [langs[i] for i in pick] + [None] * idle, num_beams, max_new_tokens, check_every,
                                      active=[1] * len(pick) + [0] * idle, track_lse=True)
            for i, k, o in zip(pick, n, res):
                if langs[i] is None:
                    langs[i] = o["language"]
                seq = o["tokens"][:-1] if o["tokens"] and o["tokens"][-1] == sp["eot"] else o["tokens"]
                skipped = o["no_speech_prob"] > NO_SPEECH_THRESHOLD and o["avg_logprob"] < LOGPROB_THRESHOLD
                kept, off = ([], k) if skipped else retrieve_segment(seq, sp["ts_begin"], k)
                windows[i].append(dict(seek=seek[i], n_frames=k, tokens=o["tokens"], kept=kept, score=o["score"],
                                       avg_logprob=o["avg_logprob"], no_speech_prob=o["no_speech_prob"], skipped=skipped,
                                       steps=steps))
                seek[i] += off
        return [dict(language=langs[i], tokens=[t for w in windows[i] for t in w["kept"]], windows=windows[i]) for i in range(P)]

    @torch.no_grad()
    def teacher_forced_logits(self, enc, tokens):
        """Decoder logits [B, T, V] of token rows [B, T] (host ints) through the decode step, one position at a time."""
        B, T = len(tokens), len(tokens[0])
        st = self._state(B, 1, enc.device)
        self.cross_kv(enc, st["ckv"])
        out = []
        for t in range(T):
            st["pos"].fill_(t)
            st["tok"].copy_(torch.tensor([r[t] for r in tokens], dtype=torch.int32))
            out.append(self._forward_rows(st).clone())
        return torch.stack(out, 1)
