"""CPU restatement of the UVR5 VR separator: CascadedASPPNet.predict (lib_v5/vr_network/nets.py, layers.py) and
SeparateVR.inference (uvr5/separate.py:198-273), in stock torch / numpy fp32, with seeded weights.

Key names are the reference's state_dict names (`stg1_low_band_net.enc1.conv1.conv.0.weight`, ...).  BatchNorm runs in eval
mode with the running statistics; every activation is ReLU except the encoders' LeakyReLU(0.01).  oracle/pin_uvr5.py checks
this file against the unmodified reference."""
import numpy as np
import torch
import torch.nn.functional as F

# get_nets_model(n_fft, size) parameter sets: (band nets nin, ch, enlarge), bridge 2 (nin, nout), full-band net 2,
# bridge 3, full-band net 3, output conv (nin, nout)
SIZES = {
    16983: dict(ch1=16, bridge2=(18, 8), ch2=16, bridge3=(34, 16), ch3=32, enlarge=False),
    33966: dict(ch1=16, bridge2=(18, 8), ch2=16, bridge3=(34, 16), ch3=32, enlarge=True),
    61968: dict(ch1=32, bridge2=(34, 16), ch2=32, bridge3=(66, 32), ch3=64, enlarge=False),
    123812: dict(ch1=32, bridge2=(34, 16), ch2=32, bridge3=(66, 32), ch3=64, enlarge=False),
    123821: dict(ch1=32, bridge2=(34, 16), ch2=32, bridge3=(66, 32), ch3=64, enlarge=False),
    537227: dict(ch1=64, bridge2=(66, 32), ch2=64, bridge3=(130, 64), ch3=128, enlarge=True),
    537238: dict(ch1=64, bridge2=(66, 32), ch2=64, bridge3=(130, 64), ch3=128, enlarge=True),
}
OFFSET = 128
DILATIONS = (4, 8, 16)


def _cbr(spec, p, nin, nout, k):
    spec[p + ".conv.0.weight"] = (nout, nin, k, k)
    for n in ("weight", "bias", "running_mean", "running_var"):
        spec[f"{p}.conv.1.{n}"] = (nout,)
    spec[p + ".conv.1.num_batches_tracked"] = ()


def _sep(spec, p, nin, nout):
    spec[p + ".conv.0.weight"] = (nin, 1, 3, 3)
    spec[p + ".conv.1.weight"] = (nout, nin, 1, 1)
    for n in ("weight", "bias", "running_mean", "running_var"):
        spec[f"{p}.conv.2.{n}"] = (nout,)
    spec[p + ".conv.2.num_batches_tracked"] = ()


def _base(spec, p, nin, ch, enlarge):
    for i, (a, b) in enumerate([(nin, ch), (ch, 2 * ch), (2 * ch, 4 * ch), (4 * ch, 8 * ch)], 1):
        _cbr(spec, f"{p}.enc{i}.conv1", a, b, 3)
        _cbr(spec, f"{p}.enc{i}.conv2", b, b, 3)
    c = 8 * ch
    _cbr(spec, f"{p}.aspp.conv1.1", c, c, 1)
    _cbr(spec, f"{p}.aspp.conv2", c, c, 1)
    for i in range(3, 6):
        _sep(spec, f"{p}.aspp.conv{i}", c, c)
    _cbr(spec, f"{p}.aspp.bottleneck.0", c * (7 if enlarge else 5), 16 * ch, 1)
    if enlarge:                     # registered after the bottleneck, which keeps its first place when reassigned
        for i in (6, 7):
            _sep(spec, f"{p}.aspp.conv{i}", c, c)
    for i, (a, b) in zip((4, 3, 2, 1), [(24 * ch, 8 * ch), (12 * ch, 4 * ch), (6 * ch, 2 * ch), (3 * ch, ch)]):
        _cbr(spec, f"{p}.dec{i}.conv", a, b, 3)


def param_spec(size=61968):
    """-> {state_dict key: shape} of get_nets_model(n_fft, size), in the reference's key order."""
    s = SIZES[size]
    spec = {}
    _base(spec, "stg1_low_band_net", 2, s["ch1"], s["enlarge"])
    _base(spec, "stg1_high_band_net", 2, s["ch1"], s["enlarge"])
    _cbr(spec, "stg2_bridge", *s["bridge2"], 1)
    _base(spec, "stg2_full_band_net", s["bridge2"][1], s["ch2"], s["enlarge"])
    _cbr(spec, "stg3_bridge", *s["bridge3"], 1)
    _base(spec, "stg3_full_band_net", s["bridge3"][1], s["ch3"], s["enlarge"])
    spec["out.weight"] = (2, s["ch3"], 1, 1)
    spec["aux1_out.weight"] = (2, s["ch1"], 1, 1)
    spec["aux2_out.weight"] = (2, s["ch2"], 1, 1)
    return spec


def init_params(spec, seed):
    """Seeded weights: He-scaled convolutions, BN affine weight in [0.5, 1.5], bias / running mean ~ N(0, 0.1^2) (not zero),
    running variance in [0.5, 2]."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for k, shape in spec.items():
        if k.endswith("num_batches_tracked"):
            P[k] = torch.tensor(0, dtype=torch.long)
        elif k.endswith(".running_var"):
            P[k] = 0.5 + 1.5 * torch.rand(shape, generator=g)
        elif k.endswith(".running_mean") or k.endswith(".bias"):
            P[k] = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:
            P[k] = 0.5 + torch.rand(shape, generator=g)
        else:
            fan_in = shape[1] * shape[2] * shape[3]
            P[k] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
    return P


def _bn_act(P, p, x, act):
    x = F.batch_norm(x, P[p + ".running_mean"], P[p + ".running_var"], P[p + ".weight"], P[p + ".bias"], False, 0.0, 1e-5)
    return F.leaky_relu(x, 0.01) if act == "lrelu" else F.relu(x)


def _cbr_f(P, p, x, stride=1, act="relu"):
    w = P[p + ".conv.0.weight"]
    return _bn_act(P, p + ".conv.1", F.conv2d(x, w, None, stride, w.shape[-1] // 2), act)


def _sep_f(P, p, x, dil):
    x = F.conv2d(x, P[p + ".conv.0.weight"], None, 1, dil, dil, groups=x.shape[1])
    return _bn_act(P, p + ".conv.2", F.conv2d(x, P[p + ".conv.1.weight"]), "relu")


def _aspp(P, p, x, enlarge):
    h, w = x.shape[2:]
    feats = [F.interpolate(_cbr_f(P, p + ".conv1.1", F.adaptive_avg_pool2d(x, (1, None))), size=(h, w), mode="bilinear",
                           align_corners=True),
             _cbr_f(P, p + ".conv2", x)]
    dils = DILATIONS + ((DILATIONS[2],) * 2 if enlarge else ())
    feats += [_sep_f(P, f"{p}.conv{i}", x, d) for i, d in zip(range(3, 8), dils)]
    return _cbr_f(P, p + ".bottleneck.0", torch.cat(feats, dim=1))


def base_net(P, p, x, enlarge):
    skips = []
    for i in range(1, 5):
        s = _cbr_f(P, f"{p}.enc{i}.conv1", x, 1, "lrelu")
        x = _cbr_f(P, f"{p}.enc{i}.conv2", s, 2, "lrelu")
        skips.append(s)
    x = _aspp(P, p + ".aspp", x, enlarge)
    for i in range(4, 0, -1):
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        x = _cbr_f(P, f"{p}.dec{i}.conv", torch.cat([x, skips[i - 1]], dim=1))
    return x


def predict(P, x_mag, aggressiveness=None, n_fft=1344, enlarge=False):
    """CascadedASPPNet(n_fft).predict in eval mode: x_mag [B, 2, n_fft // 2 + 1, W] -> [B, 2, n_fft // 2 + 1, W - 256]."""
    max_bin, out_bin = n_fft // 2, n_fft // 2 + 1
    mix = x_mag
    x = x_mag[:, :, :max_bin]
    bw = max_bin // 2
    aux1 = torch.cat([base_net(P, "stg1_low_band_net", x[:, :, :bw], enlarge),
                      base_net(P, "stg1_high_band_net", x[:, :, bw:], enlarge)], dim=2)
    aux2 = base_net(P, "stg2_full_band_net", _cbr_f(P, "stg2_bridge", torch.cat([x, aux1], dim=1)), enlarge)
    h = base_net(P, "stg3_full_band_net", _cbr_f(P, "stg3_bridge", torch.cat([x, aux1, aux2], dim=1)), enlarge)
    mask = torch.sigmoid(F.conv2d(h, P["out.weight"]))
    mask = F.pad(mask, (0, 0, 0, out_bin - mask.shape[2]), mode="replicate")
    if aggressiveness:
        sb = aggressiveness["split_bin"]
        mask[:, :, :sb] = torch.pow(mask[:, :, :sb], 1 + aggressiveness["value"] / 3)
        mask[:, :, sb:] = torch.pow(mask[:, :, sb:], 1 + aggressiveness["value"])
    return (mask * mix)[:, :, :, OFFSET:-OFFSET]


def make_padding(width, crop_size, offset):
    """-> (left, right, roi_size) of SeparateVR.make_padding"""
    left = offset
    roi = crop_size - 2 * offset
    if roi == 0:
        roi = crop_size
    return left, roi - (width % roi) + left, roi


def inference(P, x_spec, aggressiveness, data, n_fft=1344, enlarge=False):
    """SeparateVR.inference on the CPU: complex x_spec [2, n_fft // 2 + 1, n_frame] -> (pred * coef, |x|, exp(1j angle(x)))."""
    x_mag = np.abs(x_spec)
    x_phase = np.angle(x_spec)
    coef = x_mag.max()
    x_pre = x_mag / coef
    n_frame = x_pre.shape[2]
    ws = data["window_size"]
    pad_l, pad_r, roi = make_padding(n_frame, ws, OFFSET)
    n_window = int(np.ceil(n_frame / roi))

    def run(pad_l, pad_r, n_window):
        xp = np.pad(x_pre, ((0, 0), (0, 0), (pad_l, pad_r)), mode="constant")
        with torch.no_grad():
            out = [predict(P, torch.from_numpy(xp[None, :, :, i * roi: i * roi + ws]), aggressiveness, n_fft, enlarge)[0].numpy()
                   for i in range(n_window)]
        return np.concatenate(out, axis=2)

    pred = run(pad_l, pad_r, n_window)[:, :, :n_frame]
    if data["tta"]:
        pred_tta = run(pad_l + roi // 2, pad_r + roi // 2, n_window + 1)[:, :, roi // 2:][:, :, :n_frame]
        return (pred + pred_tta) * 0.5 * coef, x_mag, np.exp(1.0j * x_phase)
    return pred * coef, x_mag, np.exp(1.0j * x_phase)


def make_spec(seed, bins, n_frame):
    """Seeded stereo complex spectrogram [2, bins, n_frame] (complex64) with a decaying magnitude envelope over frequency."""
    rs = np.random.RandomState(seed)
    env = np.exp(-np.arange(bins) / (bins / 4.0))[None, :, None]
    re, im = rs.randn(2, 2, bins, n_frame)
    return ((re + 1j * im) * env).astype(np.complex64)
