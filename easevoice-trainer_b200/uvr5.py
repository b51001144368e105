"""UVR5 VR separation on the library's kernels: the CascadedASPPNet of the HP2 / HP3 / HP5 models
(lib_v5/vr_network/nets.py, layers.py), the CascadedNet of the DeEcho / DeReverb models (nets_new.py, layers_new.py; see
CascadedNet for its layout), and a batched drop-in for SeparateVR.inference (uvr5/separate.py:198-273), which
SeparateVREcho inherits.

The reference runs the net on one 512-frame window per call, copying each result to the host before the next.  Here every
window of a file, TTA windows included, goes through the net in batches of `max_windows`, and the result reaches the host
once.  Activations are channels-last fp32; a layer writes straight into its slice of the next concat buffer:
  * Encoder i's conv1 (the skip) writes channels [2 C_i, 3 C_i) of Decoder i's input, the x2 upsample of the layer below
    writes channels [0, 2 C_i);
  * the five (seven with `enlarge`) ASPP branches write slices of the bottleneck's input;
  * the input x, aux1 (the two band nets, each on its half of the rows) and aux2 are slices of one [B, max_bin, W, 2 + ...]
    buffer, so cat([x, aux1]) and cat([x, aux1, aux2]) are never built.
Eval BatchNorm is folded into a per-channel scale and bias of the preceding convolution at load; Dropout is the identity.

separate_wave runs the whole of SeparateVR.separate (uvr5/separate.py:103-196) from the decoded 44.1 kHz waveform to the two
output waveforms on the device: the band loop's polyphase resampling, the per-band STFTs written into the combined
spectrogram, the net, and per output the mask, mirroring, band filters, per-band iSTFTs and the FFT resampling that chains
the bands.  One copy to the device and one back per file.  Decoding, and resampling inputs that are not at the top band's
rate, stay with the caller.
"""
import math

import numpy as np
import torch

from . import ops
from .ops import CLView
from .weights import check_state_dict, to_device

# get_nets_model(n_fft, size) parameter sets (nets.py:125-206): band-net width, bridge 2 (nin, nout), full-band net 2
# width, bridge 3, full-band net 3 width, and whether the ASPP modules carry the two extra dilation-16 branches.
SIZES = {
    61968: dict(ch1=32, bridge2=(34, 16), ch2=32, bridge3=(66, 32), ch3=64, enlarge=False),
    123812: dict(ch1=32, bridge2=(34, 16), ch2=32, bridge3=(66, 32), ch3=64, enlarge=False),
    123821: dict(ch1=32, bridge2=(34, 16), ch2=32, bridge3=(66, 32), ch3=64, enlarge=False),
    33966: dict(ch1=16, bridge2=(18, 8), ch2=16, bridge3=(34, 16), ch3=32, enlarge=True),
    16983: dict(ch1=16, bridge2=(18, 8), ch2=16, bridge3=(34, 16), ch3=32, enlarge=False),
    537227: dict(ch1=64, bridge2=(66, 32), ch2=64, bridge3=(130, 64), ch3=128, enlarge=True),
    537238: dict(ch1=64, bridge2=(66, 32), ch2=64, bridge3=(130, 64), ch3=128, enlarge=True),
}
DILATIONS = (4, 8, 16)
BN_EPS = 1e-5


def _cbr_keys(spec, p, nin, nout, k):
    spec[p] = ("cbr", (nout, nin, k, k))


def _base_keys(spec, p, nin, ch, enlarge):
    for i, (a, b) in enumerate([(nin, ch), (ch, 2 * ch), (2 * ch, 4 * ch), (4 * ch, 8 * ch)], 1):
        _cbr_keys(spec, f"{p}.enc{i}.conv1", a, b, 3)
        _cbr_keys(spec, f"{p}.enc{i}.conv2", b, b, 3)
    c = 8 * ch
    _cbr_keys(spec, f"{p}.aspp.conv1.1", c, c, 1)
    _cbr_keys(spec, f"{p}.aspp.conv2", c, c, 1)
    for i in range(3, 8 if enlarge else 6):
        spec[f"{p}.aspp.conv{i}"] = ("sep", (c, c))
    _cbr_keys(spec, f"{p}.aspp.bottleneck.0", c * (7 if enlarge else 5), 16 * ch, 1)
    for i, (a, b) in zip((4, 3, 2, 1), [(24 * ch, 8 * ch), (12 * ch, 4 * ch), (6 * ch, 2 * ch), (3 * ch, ch)]):
        _cbr_keys(spec, f"{p}.dec{i}.conv", a, b, 3)


def layer_spec(size):
    """-> {module prefix: (kind, shape)}: "cbr" = Conv2d (no bias) + BatchNorm2d, "sep" = depthwise 3x3 + 1x1 + BatchNorm2d
    (shape (nin, nout)), "conv" = a bias-free 1x1 Conv2d"""
    s = SIZES[size]
    spec = {}
    _base_keys(spec, "stg1_low_band_net", 2, s["ch1"], s["enlarge"])
    _base_keys(spec, "stg1_high_band_net", 2, s["ch1"], s["enlarge"])
    _cbr_keys(spec, "stg2_bridge", *s["bridge2"], 1)
    _base_keys(spec, "stg2_full_band_net", s["bridge2"][1], s["ch2"], s["enlarge"])
    _cbr_keys(spec, "stg3_bridge", *s["bridge3"], 1)
    _base_keys(spec, "stg3_full_band_net", s["bridge3"][1], s["ch3"], s["enlarge"])
    spec["out"] = ("conv", (2, s["ch3"], 1, 1))
    spec["aux1_out"] = ("conv", (2, s["ch1"], 1, 1))
    spec["aux2_out"] = ("conv", (2, s["ch2"], 1, 1))
    return spec


def state_dict_shapes(size):
    """-> {state_dict key: shape} of the reference's get_nets_model(n_fft, size), num_batches_tracked left out"""
    out = {}
    for p, (kind, shape) in layer_spec(size).items():
        if kind == "conv":
            out[p + ".weight"] = shape
            continue
        if kind == "cbr":
            out[p + ".conv.0.weight"] = shape
            bn, n = p + ".conv.1", shape[0]
        else:
            nin, n = shape
            out[p + ".conv.0.weight"] = (nin, 1, 3, 3)
            out[p + ".conv.1.weight"] = (n, nin, 1, 1)
            bn = p + ".conv.2"
        for k in ("weight", "bias", "running_mean", "running_var"):
            out[f"{bn}.{k}"] = (n,)
    return out


def _fold_bn(sd, bn):
    """eval BatchNorm2d -> (scale, bias) with y = x * scale + bias, folded in float64"""
    var, mean = sd[bn + ".running_var"].double(), sd[bn + ".running_mean"].double()
    scale = sd[bn + ".weight"].double() / torch.sqrt(var + BN_EPS)
    return scale.float(), (sd[bn + ".bias"].double() - mean * scale).float()


def _cl_weight(w):
    """[N, C, k, k] -> [N, k, k, C] fp32 (the implicit GEMM's tap-major, channel-minor K order)"""
    return w.float().permute(0, 2, 3, 1).contiguous()


class _SpecNet:
    """What the two VR nets share: bins, the device, the folded layers, and the shape rules of their inputs."""

    def __init__(self, n_fft, offset):
        self.max_bin = n_fft // 2
        self.output_bin = n_fft // 2 + 1
        self.offset = offset
        self.device = torch.device("cpu")
        self.layers = None

    def to(self, device):
        self.device = torch.device(device)
        if self.layers is not None:
            self.layers = to_device(self.layers, self.device)
        return self

    def eval(self):
        return self

    def check_input(self, x, crop):
        if not (torch.is_tensor(x) and x.dim() == 4 and x.shape[1] == 2 and x.shape[2] == self.output_bin):
            raise ValueError(f"expected [B, 2, {self.output_bin}, W] magnitudes, got "
                             f"{tuple(x.shape) if torch.is_tensor(x) else type(x)}")
        self.check_shape(x.shape[3], crop)
        if self.layers is None:
            raise ValueError("no weights loaded")
        if not x.is_cuda or self.device.type != "cuda":
            raise ValueError("the VR net runs on CUDA tensors and weights only")

    def check_shape(self, W, crop):
        """The shapes the net takes: both band heights and W multiples of 16 (four stride-2 encoders, then x2 upsamples
        that must meet their skips), and W > 2 * offset when cropped.  The reference fails inside torch.cat or asserts."""
        if self.max_bin % 2 or (self.max_bin // 2) % 16:
            raise ValueError(f"band height {self.max_bin // 2} (n_fft // 4) must be a multiple of 16 and n_fft // 2 even")
        if W % 16:
            raise ValueError(f"frame count {W} must be a multiple of 16")
        if crop and W <= 2 * self.offset:
            raise ValueError(f"frame count {W} must exceed 2 * offset = {2 * self.offset}")

    def _empty(self, B, H, W, C):
        return torch.empty((B, H, W, C), device=self.device, dtype=torch.float32)

    def _conv(self, p, x, y, stride=1, act=ops.C2_RELU, dil=1):
        """folded Conv2d + BatchNorm + act of layer p; dil is an int or a (rows, columns) pair, padding = dil * (k // 2)"""
        L = self.layers[p]
        k = L["k"]
        pad = tuple(d * (k // 2) for d in dil) if isinstance(dil, tuple) else dil * (k // 2)
        ops.conv2d(x, L["w"], y, k=k, stride=stride, pad=pad, dil=dil, scale=L["scale"], bias=L["bias"], act=act)


class CascadedASPPNet(_SpecNet):
    """nets.CascadedASPPNet(n_fft, params) in eval mode on CUDA.  Input [B, 2, n_fft // 2 + 1, W] magnitudes (fp32)."""

    def __init__(self, n_fft, size=61968):
        if size not in SIZES:
            raise ValueError(f"unknown VR net size {size}; known: {sorted(SIZES)}")
        super().__init__(n_fft, 128)
        self.size, self.cfg = size, SIZES[size]

    # ---- weights -----------------------------------------------------------------------------------------
    def load_state_dict(self, sd):
        """Reference state_dict (fp16 or fp32 storage) -> folded, channels-last fp32 layers on self.device.  Keys ending in
        num_batches_tracked are ignored; any other missing or unexpected key, a non-float tensor or a wrong shape raises
        ValueError."""
        sd = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
        check_state_dict(sd, state_dict_shapes(self.size), f"CascadedASPPNet size {self.size}")
        layers = {}
        for p, (kind, shape) in layer_spec(self.size).items():
            if kind == "conv":
                layers[p] = dict(w=sd[p + ".weight"].float().reshape(shape[0], shape[1]).contiguous())
            elif kind == "cbr":
                scale, bias = _fold_bn(sd, p + ".conv.1")
                layers[p] = dict(w=_cl_weight(sd[p + ".conv.0.weight"]), scale=scale, bias=bias, k=shape[-1])
            else:
                scale, bias = _fold_bn(sd, p + ".conv.2")
                layers[p] = dict(dw=sd[p + ".conv.0.weight"].float().reshape(shape[0], 9).contiguous(),
                                 w=_cl_weight(sd[p + ".conv.1.weight"]), scale=scale, bias=bias, k=1)
        self.layers = to_device(layers, self.device)
        return self

    @classmethod
    def from_pretrained(cls, path, n_fft=1344, device="cuda"):
        """Load a VR-net .pth (HP2 / HP3 / HP5 ...): the parameter set is read from the weight shapes (band-net width from
        enc1, `enlarge` from the presence of aspp.conv6 / conv7).  Weights that match no get_nets_model set raise
        ValueError."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        return cls(n_fft, infer_size(sd)).to(device).load_state_dict(sd)

    # ---- forward -----------------------------------------------------------------------------------------
    def forward(self, x, aggressiveness=None):
        """mask * x over all W frames: [B, 2, output_bin, W] (CascadedASPPNet.forward in eval mode)"""
        self.check_input(x, crop=False)
        return self._run(x, aggressiveness, 0)

    __call__ = forward

    def predict(self, x_mag, aggressiveness=None):
        """forward cropped by `offset` frames on both time edges: [B, 2, output_bin, W - 256]"""
        self.check_input(x_mag, crop=True)
        return self._run(x_mag, aggressiveness, self.offset)

    def _aspp(self, p, x, enlarge):
        B, H, W, c = x.B, x.H, x.W, x.C
        nb = 7 if enlarge else 5
        A = self._empty(B, H, W, nb * c)
        pooled = self._empty(B, 1, W, c)
        self._conv(p + ".conv1.1", CLView(ops.mean_h(x)), CLView(pooled))
        ops.resize_bilinear_ac(CLView(pooled), CLView(A, 0, c))
        self._conv(p + ".conv2", x, CLView(A, c, c))
        dw = self._empty(B, H, W, c)
        dils = DILATIONS + ((DILATIONS[2],) * 2 if enlarge else ())
        for j, d in enumerate(dils):
            name = f"{p}.conv{3 + j}"
            ops.dwconv3x3(x, self.layers[name]["dw"], CLView(dw), d)
            self._conv(name, CLView(dw), CLView(A, (2 + j) * c, c))
        out = self._empty(B, H, W, self.layers[p + ".bottleneck.0"]["w"].shape[0])
        self._conv(p + ".bottleneck.0", CLView(A), CLView(out))
        return out

    def _base(self, p, x: CLView, out: CLView):
        """BaseASPPNet: x [B, H, W, nin] -> out [B, H, W, ch] (H, W multiples of 16)"""
        B, H, W = x.B, x.H, x.W
        ch = self.layers[p + ".enc1.conv1"]["w"].shape[0]
        dec_in, h = [], x
        for i in range(4):
            Ci, Hi, Wi = ch << i, H >> i, W >> i
            D = self._empty(B, Hi, Wi, 3 * Ci)                    # [upsampled (2 Ci) | skip (Ci)]
            skip = CLView(D, 2 * Ci, Ci)
            self._conv(f"{p}.enc{i + 1}.conv1", h, skip, act=ops.C2_LRELU)
            nxt = self._empty(B, Hi // 2, Wi // 2, Ci)
            self._conv(f"{p}.enc{i + 1}.conv2", skip, CLView(nxt), stride=2, act=ops.C2_LRELU)
            dec_in.append(D)
            h = CLView(nxt)
        h = CLView(self._aspp(p + ".aspp", h, self.cfg["enlarge"]))
        for i in range(3, -1, -1):
            D = dec_in[i]
            ops.resize_bilinear_ac(h, CLView(D, 0, 2 * (ch << i)))
            y = out if i == 0 else CLView(self._empty(B, H >> i, W >> i, ch << i))
            self._conv(f"{p}.dec{i + 1}.conv", CLView(D), y)
            h = y

    def _run(self, x, aggressiveness, offset):
        x = x.detach().float().contiguous()
        B, _, _, W = x.shape
        mb, bw = self.max_bin, self.max_bin // 2
        c1, c2 = self.cfg["ch1"], self.cfg["ch2"]
        # [x | aux1 | aux2] over all max_bin rows; the band nets read and write their own halves of the rows
        cat3 = self._empty(B, mb, W, 2 + c1 + c2)
        cat3[..., :2].copy_(x[:, :, :mb].permute(0, 2, 3, 1))
        for name, r0 in (("stg1_low_band_net", 0), ("stg1_high_band_net", bw)):
            self._base(name, CLView(cat3, 0, 2, r0, bw), CLView(cat3, 2, c1, r0, bw))
        br2 = self._empty(B, mb, W, self.cfg["bridge2"][1])
        self._conv("stg2_bridge", CLView(cat3, 0, 2 + c1), CLView(br2))
        self._base("stg2_full_band_net", CLView(br2), CLView(cat3, 2 + c1, c2))
        br3 = self._empty(B, mb, W, self.cfg["bridge3"][1])
        self._conv("stg3_bridge", CLView(cat3), CLView(br3))
        del cat3, br2
        h = self._empty(B, mb, W, self.cfg["ch3"])
        self._base("stg3_full_band_net", CLView(br3), CLView(h))
        del br3
        if aggressiveness:
            v = aggressiveness["value"]
            sb = int(aggressiveness["split_bin"])
            sb = max(0, self.output_bin + sb) if sb < 0 else min(sb, self.output_bin)   # python slice bounds
            return ops.vr_mask_head(CLView(h), self.layers["out"]["w"], x, offset, sb, 1 + v / 3, 1 + v, True)
        return ops.vr_mask_head(CLView(h), self.layers["out"]["w"], x, offset)


def infer_size(sd):
    """-> the get_nets_model size whose layers match the shapes of state_dict sd; ValueError if none does"""
    key = "stg1_low_band_net.enc1.conv1.conv.0.weight"
    if key not in sd:
        raise ValueError(f"not a VR CascadedASPPNet state_dict: no {key}")
    ch = sd[key].shape[0]
    enlarge = "stg1_low_band_net.aspp.conv6.conv.0.weight" in sd
    for size, s in SIZES.items():
        if s["ch1"] == ch and s["enlarge"] == enlarge:
            want = state_dict_shapes(size)
            have = {k: tuple(v.shape) for k, v in sd.items() if not k.endswith("num_batches_tracked")}
            if have == {k: tuple(v) for k, v in want.items()}:
                return size
    raise ValueError(f"state_dict (band width {ch}, enlarge={enlarge}) matches no get_nets_model parameter set")


def get_nets_model(n_fft, size=61968):
    """nets.get_nets_model: an unloaded CascadedASPPNet (call load_state_dict, then .to("cuda"))"""
    return CascadedASPPNet(n_fft, size)


# ---- DeEcho / DeReverb: nets_new.CascadedNet (layers_new.py) ------------------------------------------------------
ECHO_DILATIONS = ((4, 2), (8, 4), (12, 6))      # ASPP conv3..conv5, (rows, columns); padding = dilation


def _round4(c):
    return (c + 3) // 4 * 4


def _skip_first(n_up, n_skip):
    """Decoder input columns: the reference concatenates [upsampled (n_up) | skip (n_skip)]; the buffers here hold the skip
    first, so every slice an encoder writes and reads starts 16-byte aligned -> where reference channel i goes"""
    return [n_skip + i for i in range(n_up)] + list(range(n_skip))


def _echo_base_keys(spec, p, nin, ch, nin_lstm, nout_lstm):
    spec[p + ".enc1"] = ("cbr", (ch, nin, 3))
    for i, (a, b) in zip(range(2, 6), [(ch, 2 * ch), (2 * ch, 4 * ch), (4 * ch, 6 * ch), (6 * ch, 8 * ch)]):
        spec[f"{p}.enc{i}.conv1"] = ("cbr", (b, a, 3))
        spec[f"{p}.enc{i}.conv2"] = ("cbr", (b, b, 3))
    c = 8 * ch
    spec[p + ".aspp.conv1.1"] = ("cbr", (c, c, 1))
    spec[p + ".aspp.conv2"] = ("cbr", (c, c, 1))
    for i in range(3, 6):
        spec[f"{p}.aspp.conv{i}"] = ("cbr", (c, c, 3))
    spec[p + ".aspp.bottleneck"] = ("cbr", (c, 5 * c, 1))
    for i, (a, b) in zip((4, 3, 2), [(14 * ch, 6 * ch), (10 * ch, 4 * ch), (6 * ch, 2 * ch)]):
        spec[f"{p}.dec{i}.conv1"] = ("cbr", (b, a, 3))
    spec[p + ".lstm_dec2.conv"] = ("cbr", (1, 2 * ch, 1))
    spec[p + ".lstm_dec2"] = ("lstm", (nin_lstm, nout_lstm // 2))
    spec[p + ".dec1.conv1"] = ("cbr", (ch, 3 * ch + 1, 3))


def echo_layer_spec(n_fft, nout, nout_lstm=128):
    """-> {module prefix: (kind, shape)} of nets_new.CascadedNet(n_fft, nout, nout_lstm): "cbr" = Conv2d (no bias) +
    BatchNorm2d + activation, shape (nout, nin, k); "lstm" = LSTMModule's bidirectional nn.LSTM + Linear + BatchNorm1d,
    shape (bins, hidden per direction); "conv" = a bias-free 1x1 Conv2d."""
    nin_lstm = n_fft // 2 // 2
    spec = {}
    _echo_base_keys(spec, "stg1_low_band_net.0", 2, nout // 2, nin_lstm // 2, nout_lstm)
    spec["stg1_low_band_net.1"] = ("cbr", (nout // 4, nout // 2, 1))
    _echo_base_keys(spec, "stg1_high_band_net", 2, nout // 4, nin_lstm // 2, nout_lstm // 2)
    _echo_base_keys(spec, "stg2_low_band_net.0", nout // 4 + 2, nout, nin_lstm // 2, nout_lstm)
    spec["stg2_low_band_net.1"] = ("cbr", (nout // 2, nout, 1))
    _echo_base_keys(spec, "stg2_high_band_net", nout // 4 + 2, nout // 2, nin_lstm // 2, nout_lstm // 2)
    _echo_base_keys(spec, "stg3_full_band_net", 3 * nout // 4 + 2, nout, nin_lstm, nout_lstm)
    spec["out"] = ("conv", (2, nout))
    spec["aux_out"] = ("conv", (2, 3 * nout // 4))
    return spec


def echo_state_dict_shapes(n_fft, nout, nout_lstm=128):
    """-> {state_dict key: shape} of nets_new.CascadedNet(n_fft, nout, nout_lstm), num_batches_tracked left out"""
    out = {}
    for p, (kind, shape) in echo_layer_spec(n_fft, nout, nout_lstm).items():
        if kind == "conv":
            out[p + ".weight"] = shape + (1, 1)
        elif kind == "cbr":
            n, nin, k = shape
            out[p + ".conv.0.weight"] = (n, nin, k, k)
            for s in ("weight", "bias", "running_mean", "running_var"):
                out[f"{p}.conv.1.{s}"] = (n,)
        else:
            nb, hid = shape
            for d in ("", "_reverse"):
                out[f"{p}.lstm.weight_ih_l0{d}"] = (4 * hid, nb)
                out[f"{p}.lstm.weight_hh_l0{d}"] = (4 * hid, hid)
                out[f"{p}.lstm.bias_ih_l0{d}"] = (4 * hid,)
                out[f"{p}.lstm.bias_hh_l0{d}"] = (4 * hid,)
            out[p + ".dense.0.weight"] = (nb, 2 * hid)
            out[p + ".dense.0.bias"] = (nb,)
            for s in ("weight", "bias", "running_mean", "running_var"):
                out[f"{p}.dense.1.{s}"] = (nb,)
    return out


def infer_echo_config(sd):
    """-> (nout, nout_lstm) of a nets_new.CascadedNet state_dict, read from stg1_low_band_net.0's enc1 (nout // 2 rows)
    and LSTM (nout_lstm // 2 hidden units); ValueError if those keys are missing"""
    k_enc = "stg1_low_band_net.0.enc1.conv.0.weight"
    k_lstm = "stg1_low_band_net.0.lstm_dec2.lstm.weight_hh_l0"
    if k_enc not in sd or k_lstm not in sd:
        raise ValueError(f"not a DeEcho / DeReverb CascadedNet state_dict: no {k_enc if k_enc not in sd else k_lstm}")
    return 2 * sd[k_enc].shape[0], 2 * sd[k_lstm].shape[1]


class CascadedNet(_SpecNet):
    """nets_new.CascadedNet(n_fft, nout, nout_lstm) of the DeEcho / DeReverb models in eval mode on CUDA.  Input
    [B, 2, n_fft // 2 + 1, W] magnitudes (fp32).

    Layout: the input x, aux1 and aux2 are slices of one [B, max_bin, W, Cx] buffer,
    [x (2) | 0 0 | aux1 | 0.. | aux2 | 0..], so every stage input is a prefix of it whose width is a multiple of 4 (the
    wgmma path); the weights get zero columns
    for the pad channels, which are written as zeros.  A BaseNet's decoder inputs hold the encoder output (the skip) first
    and the x2 upsample after it; dec1's input is [e1 | up(dec2) | up(lstm) | 0..].  LSTMModule: the 1x1 conv gives
    [B, bins, frames] = [N][bins][T], evk_transpose_rows makes it [N][T][bins], one evk_gemm_tf32 the input projections of
    both directions (biases summed at load), evk_lstm_bidir_fwd the recurrence, one evk_gemm_tf32 the dense layer with
    BatchNorm1d folded in and ReLU, and evk_transpose_rows puts the result back as [N][bins][T], a one-channel image that
    is upsampled into its dec1 channel.  Rows of the LSTM operands are in (n, t) order throughout."""

    def __init__(self, n_fft, nout=32, nout_lstm=128):
        if nout < 4:
            raise ValueError(f"nout {nout} must be at least 4")
        if nout_lstm != 128:
            raise ValueError(f"nout_lstm {nout_lstm}: the recurrence kernel runs the hidden sizes of nout_lstm = 128 (64 and 32)")
        super().__init__(n_fft, 64)
        self.nout, self.nout_lstm = nout, nout_lstm
        self.nin_lstm = self.max_bin // 2
        q, h = nout // 4, nout // 2
        # aux1 at [4, 4 + q), aux2 at [_a2, _a2 + h); stage 2 reads [0, _a2), stage 3 [0, _cx)
        self._a2 = _round4(4 + q)
        self._cx = _round4(self._a2 + h)
        self._x_pads = [(2, 4), (4 + q, self._a2), (self._a2 + h, self._cx)]

    # ---- weights -----------------------------------------------------------------------------------------
    def _placements(self):
        """-> {layer prefix: (input column of each reference input channel, input width)} for the layers whose input is
        laid out differently from the reference's concatenation"""
        q, h = self.nout // 4, self.nout // 2
        x_cols = [0, 1]
        stage_in = {"stg1_low_band_net.0": (x_cols, 4), "stg1_high_band_net": (x_cols, 4),
                    "stg2_low_band_net.0": (x_cols + list(range(4, 4 + q)), self._a2),
                    "stg2_high_band_net": (x_cols + list(range(4, 4 + q)), self._a2),
                    "stg3_full_band_net": (x_cols + list(range(4, 4 + q)) + list(range(self._a2, self._a2 + h)), self._cx)}
        out = {}
        for p, cin in stage_in.items():
            ch = {"stg1_low_band_net.0": h, "stg1_high_band_net": q, "stg2_low_band_net.0": self.nout,
                  "stg2_high_band_net": h, "stg3_full_band_net": self.nout}[p]
            out[p + ".enc1"] = cin
            out[p + ".dec4.conv1"] = (_skip_first(8 * ch, 6 * ch), 14 * ch)
            out[p + ".dec3.conv1"] = (_skip_first(6 * ch, 4 * ch), 10 * ch)
            out[p + ".dec2.conv1"] = (_skip_first(4 * ch, 2 * ch), 6 * ch)
            out[p + ".dec1.conv1"] = (_skip_first(2 * ch + 1, ch), _round4(3 * ch + 1))
        return out

    def load_state_dict(self, sd):
        """Reference state_dict (fp16 or fp32 storage) -> folded, channels-last fp32 layers on self.device.  Keys ending in
        num_batches_tracked are ignored; any other missing or unexpected key, a non-float tensor or a wrong shape raises
        ValueError."""
        sd = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
        check_state_dict(sd, echo_state_dict_shapes(2 * self.max_bin, self.nout, self.nout_lstm),
                         f"CascadedNet(n_fft={2 * self.max_bin}, nout={self.nout}, nout_lstm={self.nout_lstm})")
        place = self._placements()
        layers = {}
        for p, (kind, shape) in echo_layer_spec(2 * self.max_bin, self.nout, self.nout_lstm).items():
            if kind == "conv":
                layers[p] = dict(w=sd[p + ".weight"].float().reshape(shape).contiguous())
            elif kind == "cbr":
                scale, bias = _fold_bn(sd, p + ".conv.1")
                w = sd[p + ".conv.0.weight"]
                if p in place:
                    cols, C = place[p]
                    wl = torch.zeros((w.shape[0], w.shape[2], w.shape[3], C), dtype=torch.float32)
                    wl[..., cols] = w.float().permute(0, 2, 3, 1)
                else:
                    wl = _cl_weight(w)
                layers[p] = dict(w=wl.contiguous(), scale=scale, bias=bias, k=shape[2])
            else:
                q = p + ".lstm."
                d = ("", "_reverse")
                w_ih = torch.cat([sd[q + "weight_ih_l0" + s].float() for s in d], 0)
                b = torch.cat([(sd[q + "bias_ih_l0" + s].double() + sd[q + "bias_hh_l0" + s].double()).float() for s in d])
                w_hh = torch.stack([sd[q + "weight_hh_l0" + s].float() for s in d])
                bn = p + ".dense.1"
                var, mean = sd[bn + ".running_var"].double(), sd[bn + ".running_mean"].double()
                sc = sd[bn + ".weight"].double() / torch.sqrt(var + BN_EPS)
                w_d = (sd[p + ".dense.0.weight"].double() * sc[:, None]).float()
                b_d = ((sd[p + ".dense.0.bias"].double() - mean) * sc + sd[bn + ".bias"].double()).float()
                layers[p] = dict(w_ih=w_ih.contiguous(), b=b, w_hh=w_hh.contiguous(), w_d=w_d.contiguous(), b_d=b_d)
        self.layers = to_device(layers, self.device)
        return self

    @classmethod
    def from_pretrained(cls, path, n_fft=1344, device="cuda"):
        """Load a DeEcho / DeReverb .pth: nout and nout_lstm are read from the weight shapes (64 for DeReverb, 48 for the
        DeEcho models).  Weights that do not form a CascadedNet at this n_fft raise ValueError."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        return cls(n_fft, *infer_echo_config(sd)).to(device).load_state_dict(sd)

    # ---- forward -----------------------------------------------------------------------------------------
    def forward(self, x):
        """the mask [B, 2, output_bin, W] over all W frames (CascadedNet.forward in eval mode)"""
        self.check_input(x, crop=False)
        return self._run(x, torch.ones_like(x), 0)

    __call__ = forward

    def predict(self, x_mag, aggressiveness=None):
        """x_mag * mask cropped by `offset` frames on both time edges: [B, 2, output_bin, W - 128].  `aggressiveness` is
        accepted and ignored, as in the reference."""
        self.check_input(x_mag, crop=True)
        return self._run(x_mag, None, self.offset)

    def _lstm(self, p, h: CLView):
        """LSTMModule: dec2's output h [B, bins, T, 2 ch] -> [B, bins, T, 1]"""
        L = self.layers[p]
        B, nb, T = h.B, h.H, h.W
        m = self._empty(B, nb, T, 1)
        self._conv(p + ".conv", h, CLView(m))
        g = ops.gemm_tf32(ops.transpose_rows(m.view(B, nb, T)).view(B * T, nb), L["w_ih"], bias=L["b"])
        y = ops.lstm_bidir(g.view(B, T, -1), L["w_hh"], order="nt")
        d = ops.gemm_tf32(y.view(B * T, -1), L["w_d"], bias=L["b_d"], act=ops.ACT_RELU)
        out = self._empty(B, nb, T, 1)
        ops.transpose_rows(d.view(B, T, nb), out=out.view(B, nb, T))
        return out

    def _aspp(self, p, x: CLView):
        B, H, W, c = x.B, x.H, x.W, x.C
        A = self._empty(B, H, W, 5 * c)
        pooled = self._empty(B, 1, W, c)
        self._conv(p + ".conv1.1", CLView(ops.mean_h(x)), CLView(pooled))
        ops.resize_bilinear_ac(CLView(pooled), CLView(A, 0, c))
        self._conv(p + ".conv2", x, CLView(A, c, c))
        for j, d in enumerate(ECHO_DILATIONS):
            self._conv(f"{p}.conv{3 + j}", x, CLView(A, (2 + j) * c, c), dil=d)
        out = self._empty(B, H, W, c)
        self._conv(p + ".bottleneck", CLView(A), CLView(out))
        return out

    def _base(self, p, x: CLView, out: CLView):
        """BaseNet: x [B, H, W, nin] -> out [B, H, W, ch] (H, W multiples of 16)"""
        B, H, W = x.B, x.H, x.W
        ch = self.layers[p + ".enc1"]["w"].shape[0]
        D1 = self._empty(B, H, W, _round4(3 * ch + 1))        # [e1 | up(dec2) | up(lstm) | 0..]
        D1[..., 3 * ch + 1:].zero_()
        self._conv(p + ".enc1", x, CLView(D1, 0, ch))
        dec_in, h = [D1], CLView(D1, 0, ch)
        for i, (cs, cu) in zip(range(2, 5), [(2 * ch, 4 * ch), (4 * ch, 6 * ch), (6 * ch, 8 * ch)]):
            s = i - 1
            t = self._empty(B, H >> s, W >> s, cs)
            self._conv(f"{p}.enc{i}.conv1", h, CLView(t), stride=2, act=ops.C2_LRELU)
            D = self._empty(B, H >> s, W >> s, cs + cu)          # [e_i | up(dec_{i+1})]
            self._conv(f"{p}.enc{i}.conv2", CLView(t), CLView(D, 0, cs), act=ops.C2_LRELU)
            dec_in.append(D)
            h = CLView(D, 0, cs)
        t = self._empty(B, H >> 4, W >> 4, 8 * ch)
        self._conv(p + ".enc5.conv1", h, CLView(t), stride=2, act=ops.C2_LRELU)
        e5 = self._empty(B, H >> 4, W >> 4, 8 * ch)
        self._conv(p + ".enc5.conv2", CLView(t), CLView(e5), act=ops.C2_LRELU)
        h = CLView(self._aspp(p + ".aspp", CLView(e5)))
        for i in (4, 3, 2):
            D = dec_in[i - 1]
            cs = (2 * ch, 4 * ch, 6 * ch)[i - 2]
            ops.resize_bilinear_ac(h, CLView(D, cs))
            y = self._empty(B, H >> (i - 1), W >> (i - 1), self.layers[f"{p}.dec{i}.conv1"]["w"].shape[0])
            self._conv(f"{p}.dec{i}.conv1", CLView(D), CLView(y))
            h = CLView(y)
        lstm = self._lstm(p + ".lstm_dec2", h)
        ops.resize_bilinear_ac(h, CLView(D1, ch, 2 * ch))
        ops.resize_bilinear_ac(CLView(lstm), CLView(D1, 3 * ch, 1))
        self._conv(p + ".dec1.conv1", CLView(D1), out)

    def _run(self, x, mix, offset):
        """mask * mix (x when mix is None), cropped by offset frames"""
        x = x.detach().float().contiguous()
        B, _, _, W = x.shape
        mb, bw = self.max_bin, self.max_bin // 2
        q, h, a2 = self.nout // 4, self.nout // 2, self._a2
        X = self._empty(B, mb, W, self._cx)                     # [x | 0 0 | aux1 | 0.. | aux2 | 0..]
        X[..., :2].copy_(x[:, :, :mb].permute(0, 2, 3, 1))
        for c0, c1 in self._x_pads:
            X[..., c0:c1].zero_()
        t = self._empty(B, bw, W, h)
        self._base("stg1_low_band_net.0", CLView(X, 0, 4, 0, bw), CLView(t))
        self._conv("stg1_low_band_net.1", CLView(t), CLView(X, 4, q, 0, bw))
        self._base("stg1_high_band_net", CLView(X, 0, 4, bw, bw), CLView(X, 4, q, bw, bw))
        t = self._empty(B, bw, W, self.nout)
        self._base("stg2_low_band_net.0", CLView(X, 0, a2, 0, bw), CLView(t))
        self._conv("stg2_low_band_net.1", CLView(t), CLView(X, a2, h, 0, bw))
        self._base("stg2_high_band_net", CLView(X, 0, a2, bw, bw), CLView(X, a2, h, bw, bw))
        del t
        f3 = self._empty(B, mb, W, self.nout)
        self._base("stg3_full_band_net", CLView(X), CLView(f3))
        del X
        return ops.vr_mask_head(CLView(f3), self.layers["out"]["w"], x if mix is None else mix.detach().float().contiguous(),
                                offset)


def make_padding(width, crop_size, offset):
    """SeparateVR.make_padding -> (left, right, roi_size)"""
    left = offset
    roi_size = crop_size - left * 2
    if roi_size == 0:
        roi_size = crop_size
    return left, roi_size - (width % roi_size) + left, roi_size


def _windows(x_pre, pad_l, pad_r, roi, ws, n_window):
    """[n_window, 2, bins, ws] windows of the zero-padded magnitudes, start i * roi (the reference's slices)"""
    xp = torch.nn.functional.pad(x_pre, (pad_l, pad_r))
    return xp.unfold(2, ws, roi)[:, :, :n_window].permute(2, 0, 1, 3)


def _predict_windows(x_pre, model, aggressiveness, ws, tta, max_windows):
    """The net over every window (and TTA window) of the normalised magnitudes x_pre [2, bins, n_frame] (device), in batches
    of max_windows -> (output [n_window (+ n_window + 1), 2, bins, roi] on the device, n_window, roi)"""
    n_frame = x_pre.shape[2]
    pad_l, pad_r, roi = make_padding(n_frame, ws, model.offset)
    n_window = int(np.ceil(n_frame / roi))
    wins = [_windows(x_pre, pad_l, pad_r, roi, ws, n_window)]
    if tta:
        wins.append(_windows(x_pre, pad_l + roi // 2, pad_r + roi // 2, roi, ws, n_window + 1))
    wins = torch.cat(wins, 0)
    outs = [model.predict(wins[i:i + max_windows].contiguous(), aggressiveness) for i in range(0, wins.shape[0], max_windows)]
    return torch.cat(outs, 0), n_window, roi


def inference(x_spec, device, model, aggressiveness, data, max_windows=16):
    """SeparateVR.inference(x_spec, device, model, aggressiveness, data) with every window (and TTA window) of the file in
    batches of max_windows: -> numpy (pred * coef, |x_spec|, exp(1j * angle(x_spec))).  |x|, the phase and coef are the
    reference's numpy computations; an all-zero spectrum gives coef = 0 and, as in the reference, a NaN pred (0 / 0)."""
    if max_windows < 1:
        raise ValueError("max_windows must be >= 1")
    ws = data["window_size"]
    if x_spec.ndim != 3 or x_spec.shape[:2] != (2, model.output_bin):
        raise ValueError(f"expected a [2, {model.output_bin}, n_frame] spectrogram, got {x_spec.shape}")
    model.check_shape(ws, crop=True)
    x_mag = np.abs(x_spec)
    coef = x_mag.max()
    x_mag_pre = x_mag / coef
    n_frame = x_mag_pre.shape[2]
    x_pre = torch.from_numpy(np.ascontiguousarray(x_mag_pre, dtype=np.float32)).to(torch.device(device))
    out, n_window, roi = _predict_windows(x_pre, model, aggressiveness, ws, data["tta"], max_windows)
    phase = np.exp(1.0j * np.angle(x_spec))                # host work while the device runs the net
    out = out.cpu().numpy()                                # the one copy to the host
    bins = out.shape[2]

    def join(o):
        return o.transpose(1, 2, 0, 3).reshape(2, bins, -1)

    pred = join(out[:n_window])[:, :, :n_frame]
    if data["tta"]:
        pred_tta = join(out[n_window:])[:, :, roi // 2:][:, :, :n_frame]
        return (pred + pred_tta) * 0.5 * coef, x_mag, phase
    return pred * coef, x_mag, phase


# ---- SeparateVR.separate from waveform to waveform -----------------------------------------------------------------
WINDOW_SIZE = 512          # SeparateVR's data["window_size"]
ZERO_PAD = True            # librosa 0.9's stft pad_mode default "constant" (unverified against a run of librosa 0.9.2)


def stft_size_ok(n_fft):
    """the frame sizes of the mixed-radix STFT core: even divisors of 61440 = 2^12 3 5 in [16, 7680]"""
    return 16 <= n_fft <= 7680 and n_fft % 2 == 0 and 61440 % n_fft == 0


def firwin_kaiser(numtaps, cutoff, beta=5.0):
    """scipy.signal.firwin(numtaps, cutoff, window=("kaiser", beta)) (low-pass, scaled to unit gain at DC), float64"""
    m = np.arange(numtaps) - (numtaps - 1) / 2.0
    h = cutoff * np.sinc(cutoff * m)
    alpha = (numtaps - 1) / 2.0
    h = h * (np.i0(beta * np.sqrt(1.0 - ((np.arange(numtaps) - alpha) / alpha) ** 2)) / np.i0(beta))
    return h / h.sum()


def poly_filter(up, down):
    """scipy.signal.resample_poly's default filter for (up, down) (already reduced): -> (the zero-prefixed fp32 taps times up,
    half_len, n_pre_remove)"""
    max_rate = max(up, down)
    half_len = 10 * max_rate
    h = firwin_kaiser(2 * half_len + 1, 1.0 / max_rate).astype(np.float32) * np.float32(up)
    n_pre_pad = down - half_len % down
    return np.concatenate([np.zeros(n_pre_pad, np.float32), h]), half_len, (half_len + n_pre_pad) // down


def lp_gains(g, bin_start, bin_stop):
    """spec_utils.fft_lp_filter applied to the per-bin gain vector g (float64)"""
    v = 1.0
    for b in range(bin_start, bin_stop):
        v -= 1 / (bin_stop - bin_start)
        g[b] = v * g[b]
    g[bin_stop:] *= 0
    return g


def hp_gains(g, bin_start, bin_stop):
    """spec_utils.fft_hp_filter applied to the per-bin gain vector g (float64)"""
    v = 1.0
    for b in range(bin_start, bin_stop, -1):
        v -= 1 / (bin_start - bin_stop)
        g[b] = v * g[b]
    g[0:bin_stop + 1] *= 0
    return g


def band_gains(param):
    """-> {band: float64 [n_fft/2 + 1]}: the filters cmb_spectrogram_to_wave applies to each band (spec_utils.py:356-431)"""
    n = len(param["band"])
    out = {}
    for d in range(1, n + 1):
        bp = param["band"][d]
        g = np.ones(bp["n_fft"] // 2 + 1)
        if d == n:
            if bp["hpf_start"] > 0:
                hp_gains(g, bp["hpf_start"], bp["hpf_stop"] - 1)
        elif d == 1:
            lp_gains(g, bp["lpf_start"], bp["lpf_stop"])
        else:
            hp_gains(g, bp["hpf_start"], bp["hpf_stop"] - 1)
            lp_gains(g, bp["lpf_start"], bp["lpf_stop"])
        out[d] = g
    return out


def pre_filter_gains(param):
    """-> float32 [bins + 1]: the row gains of combine_spectrograms' pre-filter (1 elsewhere)"""
    g = np.ones(param["bins"] + 1, np.float32)
    if param["pre_filter_start"] > 0:
        if len(param["band"]) == 1:
            raise ValueError("single-band parameter sets (fft_lp_filter pre-filter) are not supported")
        gp = 1
        for b in range(param["pre_filter_start"] + 1, param["pre_filter_stop"]):
            v = math.pow(10, -(b - param["pre_filter_start"]) * (3.5 - gp) / 20.0)
            gp = v
            g[b] = np.float32(v)
    return g


def high_end_head(param):
    """SeparateVR.separate's input_high_end_h: the number of top-band bins `mirroring` replaces"""
    bp = param["band"][len(param["band"])]
    return (bp["n_fft"] // 2 - bp["crop_stop"]) + (param["pre_filter_stop"] - param["pre_filter_start"])


def check_wave_param(param, high_end_process="mirroring"):
    """ValueError unless separate_wave can run this ModelParameters.param (see separate_wave)"""
    if high_end_process not in ("mirroring", "none"):
        raise ValueError(f"high_end_process {high_end_process!r}: only 'mirroring' and 'none' are supported")
    for k in ("mid_side", "mid_side_b2", "reverse"):
        if param.get(k):
            raise ValueError(f"parameter sets with {k} are not supported")
    bands = param["band"]
    n = len(bands)
    if sorted(bands) != list(range(1, n + 1)):
        raise ValueError("band keys must be the integers 1 .. n")
    if n > 4:
        raise ValueError(f"{n} bands: at most 4 are supported")
    if n == 1:
        raise ValueError("single-band parameter sets are not supported")
    if bands[n]["sr"] != param["sr"]:
        raise ValueError(f"top band rate {bands[n]['sr']} differs from the parameter set's sr {param['sr']}")
    for d in range(1, n + 1):
        bp = bands[d]
        if not stft_size_ok(bp["n_fft"]):
            raise ValueError(f"band {d}: n_fft {bp['n_fft']} is not an even divisor of 61440 (2^12 3 5) in [16, 7680]")
        if not 0 < bp["hl"] <= bp["n_fft"] // 2:
            raise ValueError(f"band {d}: hop {bp['hl']} must be in (0, n_fft / 2]")
        if d < n:
            up_sr = bands[d + 1]["sr"]
            if bp["res_type"] != "polyphase" or up_sr % bp["sr"]:
                raise ValueError(f"band {d}: only polyphase resampling by an integer factor is supported "
                                 f"({bp['res_type']}, {up_sr} -> {bp['sr']})")
            if bp["hl"] * up_sr != bands[d + 1]["hl"] * bp["sr"]:
                raise ValueError(f"band {d}: hop {bp['hl']} at {bp['sr']} Hz does not cover the time of band {d + 1}'s hop")
    if n > 1 and bands[1]["sr"] != bands[2]["sr"]:
        raise ValueError("the back end's sinc_fastest step between bands 1 and 2 needs equal rates")
    if sum(b["crop_stop"] - b["crop_start"] for b in bands.values()) > param["bins"]:
        raise ValueError("Too much bins")
    if high_end_process == "mirroring" and param["pre_filter_start"] - 10 - high_end_head(param) < 0:
        raise ValueError("the mirrored rows start before row 0")


def resampled_len(n, orig_sr, target_sr):
    """librosa.resample's output length: n for equal rates, else int(ceil(n * (target_sr / orig_sr))) in float64 (fix_length
    pads or trims scipy's output to it)"""
    return n if orig_sr == target_sr else int(np.ceil(n * (float(target_sr) / orig_sr)))


def band_lengths(L, param):
    """-> {band: samples} down the band loop from L samples at the top band"""
    bands = param["band"]
    n = len(bands)
    out = {n: L}
    for d in range(n - 1, 0, -1):
        out[d] = resampled_len(out[d + 1], bands[d + 1]["sr"], bands[d]["sr"])
    return out


def fft_resample(x, num):
    """scipy.signal.resample(x, num, axis=-1) of float64 rows x [rows, Nx].  One transform of an arbitrary length (80 (l - 1)
    samples at 7350 Hz, with factors such as 23 * 719) per band boundary: torch.fft's, a few milliseconds against the
    net's hundreds."""
    Nx = x.shape[-1]
    X = torch.fft.rfft(x, dim=-1)
    Y = torch.zeros(x.shape[:-1] + (num // 2 + 1,), dtype=X.dtype, device=x.device)
    N = min(num, Nx)
    nyq = N // 2 + 1
    Y[..., :nyq] = X[..., :nyq]
    if N % 2 == 0:
        if num < Nx:
            Y[..., N // 2] *= 2.0
        elif Nx < num:
            Y[..., N // 2] *= 0.5
    return torch.fft.irfft(Y, n=num, dim=-1) * (float(num) / float(Nx))


def separate_wave(wave, model, param, agg=10, tta=False, high_end_process="mirroring", max_windows=16):
    """SeparateVR.separate (and SeparateVREcho's) from the decoded waveform to the two output waveforms, on the device:
    -> (accompaniment, vocals), numpy float32 [hop_top * (l - 1), 2] each: the wav_accompaniment and wav_vocals of
    separate.py:165-187 before `* 32768` and the int16 cast.

    wave: float32 [2, L] or [L] (mono is duplicated) at the top band's rate, param["sr"].  param: ModelParameters.param (int
    band keys), e.g. 4band_v2 (SeparateVR) or 4band_v3 (SeparateVREcho).  model: a CascadedASPPNet or CascadedNet on CUDA.
    Parameter sets this path cannot take raise ValueError before any device work: mid_side / mid_side_b2 / reverse; a lower
    band that is not a polyphase resampling by an integer factor; different rates at the back end's sinc_fastest step; an
    n_fft that is not an even divisor of 61440 (2^12 3 5) in [16, 7680]; a top band rate other than param["sr"]; and
    high_end_process other than "mirroring" / "none".  So do inputs too short for two frames of every band.  Where the
    reference reads memory it never wrote (cmb_spectrogram_to_wave's np.ndarray: band 1's bins past crop_stop, the top
    band's Nyquist bin), zeros are used.  An all-zero input gives NaN outputs, as the reference's 0 / 0."""
    check_wave_param(param, high_end_process)
    if max_windows < 1:
        raise ValueError("max_windows must be >= 1")
    if model.output_bin != param["bins"] + 1:
        raise ValueError(f"the model has {model.output_bin} bins, the parameter set {param['bins'] + 1}")
    wave = np.asarray(wave, dtype=np.float32)
    if wave.ndim == 1:
        wave = np.stack([wave, wave])
    if wave.ndim != 2 or wave.shape[0] != 2:
        raise ValueError(f"expected a [2, L] or [L] waveform, got {wave.shape}")
    bands = param["band"]
    n = len(bands)
    lens = band_lengths(wave.shape[1], param)
    l = min(1 + lens[d] // bands[d]["hl"] for d in bands)
    if min(lens.values()) < 1 or l < 2:
        raise ValueError(f"{wave.shape[1]} samples: too short for two frames of every band")
    model.check_shape(WINDOW_SIZE, crop=True)
    dev = model.device
    # every band's two rows in one buffer; a band at the rate of the band above it is that band's rows
    offs, total = {}, 0
    for d in range(n, 0, -1):
        if d < n and bands[d]["sr"] == bands[d + 1]["sr"]:
            offs[d] = offs[d + 1]
        else:
            offs[d], total = total, total + 2 * lens[d]
    buf = torch.empty(total, device=dev, dtype=torch.float32)
    buf[offs[n]:offs[n] + 2 * lens[n]].copy_(torch.from_numpy(np.ascontiguousarray(wave)).view(-1))      # the one copy in
    for d in range(n - 1, 0, -1):
        if offs[d] != offs[d + 1]:
            g = math.gcd(bands[d + 1]["sr"], bands[d]["sr"])
            up, down = bands[d]["sr"] // g, bands[d + 1]["sr"] // g
            h, _, n_pre_remove = poly_filter(up, down)
            dst = buf[offs[d]:offs[d] + 2 * lens[d]].view(2, lens[d])
            n_poly = min(-(-lens[d + 1] * up // down), lens[d])          # resample_poly's outputs, then fix_length's zeros
            dst[:, n_poly:].zero_()
            ops.resample_poly(buf[offs[d + 1]:offs[d + 1] + 2 * lens[d + 1]].view(2, lens[d + 1]), torch.from_numpy(h).to(dev), up,
                              down, n_pre_remove, n_poly, out=dst[:, :n_poly])
    rows, row0 = param["bins"] + 1, 0
    stft_bands, asm_bands = [], []
    for d in range(1, n + 1):
        bp = bands[d]
        stft_bands.append((offs[d], lens[d], lens[d], bp["n_fft"], bp["hl"], bp["crop_start"], bp["crop_stop"], row0))
        asm_bands.append((bp["n_fft"], bp["crop_start"], bp["crop_stop"], row0))
        row0 += bp["crop_stop"] - bp["crop_start"]
    mirror = high_end_process == "mirroring"
    hh = high_end_head(param) if mirror else 0
    top = bands[n]
    x, high = ops.vr_band_stft(buf, stft_bands, l, torch.from_numpy(pre_filter_gains(param)).to(dev), rows,
                               high_band=n - 1 if mirror else -1, high_lo=top["n_fft"] // 2 - hh, high_h=hh, zero_pad=ZERO_PAD)
    del buf
    x_pre, coef = ops.vr_mag_norm(x)
    aggressiveness = {"value": float(agg / 100), "split_bin": bands[1]["crop_stop"], "aggr_correction": param.get("aggr_correction")}
    out, n_window, roi = _predict_windows(x_pre, model, aggressiveness, WINDOW_SIZE, tta, max_windows)
    del x_pre

    def join(o, skip):
        return o.permute(1, 2, 0, 3).reshape(2, rows, -1)[:, :, skip:skip + l].contiguous()

    pred = join(out[:n_window], 0)
    pred_tta = join(out[n_window:], roi // 2) if tta else None
    del out
    gains = [torch.from_numpy(g.astype(np.float32)).to(dev) for g in band_gains(param).values()]
    frames = ops.vr_assemble(x, pred, pred_tta, coef, asm_bands, gains, high=high,
                             mirror_lo=param["pre_filter_start"] - 10 - hh, top=n - 1)
    wav = None
    for d in range(1, n + 1):
        bp = bands[d]
        w = ops.istft(frames[d - 1], 4, 1, bp["n_fft"], bp["hl"]).double()
        frames[d - 1] = None
        wav = w if wav is None else wav + w
        if d < n and bands[d + 1]["sr"] != bp["sr"]:
            wav = fft_resample(wav, resampled_len(wav.shape[1], bp["sr"], bands[d + 1]["sr"]))
    res = wav.float().cpu().numpy()                                                           # the one copy out
    return np.ascontiguousarray(res[0:2].T), np.ascontiguousarray(res[2:4].T)
