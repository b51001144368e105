"""CPU restatement of the UVR5 DeEcho / DeReverb separator: CascadedNet.predict (lib_v5/vr_network/nets_new.py,
layers_new.py) and the SeparateVR.inference window loop that SeparateVREcho inherits (uvr5/separate.py:198-299), in stock
torch / numpy fp32 (F.conv2d, torch.nn.LSTM), with seeded weights.

Key names are the reference's state_dict names (`stg1_low_band_net.0.enc1.conv.0.weight`, ...).  BatchNorm runs in eval mode
with the running statistics; Dropout is the identity.  Activations: ReLU everywhere except the encoders' LeakyReLU(0.01).
`predict` ignores `aggressiveness`, as the reference's does.  oracle/pin_uvr5_echo.py checks this file against the
unmodified reference."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.uvr5_oracle import make_padding, make_spec  # noqa: F401  (same window arithmetic and test spectra)

OFFSET = 64
DILATIONS = ((4, 2), (8, 4), (12, 6))          # ASPP conv3..conv5: (rows, columns), padding = dilation
LSTM_SUFFIXES = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")


def _cbr(spec, p, nin, nout, k):
    spec[p + ".conv.0.weight"] = (nout, nin, k, k)
    for n in ("weight", "bias", "running_mean", "running_var"):
        spec[f"{p}.conv.1.{n}"] = (nout,)
    spec[p + ".conv.1.num_batches_tracked"] = ()


def _base(spec, p, nin, ch, nin_lstm, nout_lstm):
    _cbr(spec, f"{p}.enc1", nin, ch, 3)
    for i, (a, b) in zip(range(2, 6), [(ch, 2 * ch), (2 * ch, 4 * ch), (4 * ch, 6 * ch), (6 * ch, 8 * ch)]):
        _cbr(spec, f"{p}.enc{i}.conv1", a, b, 3)
        _cbr(spec, f"{p}.enc{i}.conv2", b, b, 3)
    c = 8 * ch
    _cbr(spec, f"{p}.aspp.conv1.1", c, c, 1)
    _cbr(spec, f"{p}.aspp.conv2", c, c, 1)
    for i in range(3, 6):
        _cbr(spec, f"{p}.aspp.conv{i}", c, c, 3)
    _cbr(spec, f"{p}.aspp.bottleneck", 5 * c, c, 1)
    for i, (a, b) in zip((4, 3, 2), [(14 * ch, 6 * ch), (10 * ch, 4 * ch), (6 * ch, 2 * ch)]):
        _cbr(spec, f"{p}.dec{i}.conv1", a, b, 3)
    q = f"{p}.lstm_dec2"
    _cbr(spec, q + ".conv", 2 * ch, 1, 1)
    hid = nout_lstm // 2
    for sfx in ("", "_reverse"):
        for name, shape in zip(LSTM_SUFFIXES, [(4 * hid, nin_lstm), (4 * hid, hid), (4 * hid,), (4 * hid,)]):
            spec[f"{q}.lstm.{name}{sfx}"] = shape
    spec[q + ".dense.0.weight"] = (nin_lstm, nout_lstm)
    spec[q + ".dense.0.bias"] = (nin_lstm,)
    for n in ("weight", "bias", "running_mean", "running_var"):
        spec[f"{q}.dense.1.{n}"] = (nin_lstm,)
    spec[q + ".dense.1.num_batches_tracked"] = ()
    _cbr(spec, f"{p}.dec1.conv1", 3 * ch + 1, ch, 3)


def param_spec(n_fft, nout=32, nout_lstm=128):
    """-> {state_dict key: shape} of CascadedNet(n_fft, nout, nout_lstm), in the reference's key order."""
    nin_lstm = n_fft // 2 // 2
    spec = {}
    _base(spec, "stg1_low_band_net.0", 2, nout // 2, nin_lstm // 2, nout_lstm)
    _cbr(spec, "stg1_low_band_net.1", nout // 2, nout // 4, 1)
    _base(spec, "stg1_high_band_net", 2, nout // 4, nin_lstm // 2, nout_lstm // 2)
    _base(spec, "stg2_low_band_net.0", nout // 4 + 2, nout, nin_lstm // 2, nout_lstm)
    _cbr(spec, "stg2_low_band_net.1", nout, nout // 2, 1)
    _base(spec, "stg2_high_band_net", nout // 4 + 2, nout // 2, nin_lstm // 2, nout_lstm // 2)
    _base(spec, "stg3_full_band_net", 3 * nout // 4 + 2, nout, nin_lstm, nout_lstm)
    spec["out.weight"] = (2, nout, 1, 1)
    spec["aux_out.weight"] = (2, 3 * nout // 4, 1, 1)
    return spec


def init_params(spec, seed):
    """Seeded weights: He-scaled convolutions and dense layers, BN affine weight in [0.5, 1.5], BN bias / running mean
    ~ N(0, 0.1^2) (not zero), running variance in [0.5, 2]; LSTM weights and biases U(-1/sqrt(H), 1/sqrt(H)) as
    nn.LSTM initialises them."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for k, shape in spec.items():
        if k.endswith("num_batches_tracked"):
            P[k] = torch.tensor(0, dtype=torch.long)
        elif ".lstm." in k:
            hid = shape[0] // 4
            P[k] = (torch.rand(shape, generator=g) * 2 - 1) / hid ** 0.5
        elif k.endswith(".running_var"):
            P[k] = 0.5 + 1.5 * torch.rand(shape, generator=g)
        elif k.endswith(".running_mean") or k.endswith(".bias"):
            P[k] = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:
            P[k] = 0.5 + torch.rand(shape, generator=g)
        else:
            fan_in = int(np.prod(shape[1:]))
            P[k] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
    return P


def _bn(P, p, x):
    return F.batch_norm(x, P[p + ".running_mean"], P[p + ".running_var"], P[p + ".weight"], P[p + ".bias"], False, 0.0, 1e-5)


def _cbr_f(P, p, x, stride=1, act="relu", dil=(1, 1)):
    w = P[p + ".conv.0.weight"]
    k = w.shape[-1]
    pad = (dil[0] * (k // 2), dil[1] * (k // 2))
    x = _bn(P, p + ".conv.1", F.conv2d(x, w, None, stride, pad, dil))
    return F.leaky_relu(x, 0.01) if act == "lrelu" else F.relu(x)


def lstm_modules(P, device="cpu", dtype=torch.float32):
    """-> {LSTMModule prefix: torch.nn.LSTM holding P's weights} (built once; predict(..., lstms=) reuses them)"""
    out = {}
    for k in P:
        if k.endswith(".lstm.weight_hh_l0"):
            p = k[: -len(".weight_hh_l0")]
            hid, nin = P[k].shape[1], P[p + ".weight_ih_l0"].shape[1]
            m = torch.nn.LSTM(nin, hid, bidirectional=True)
            with torch.no_grad():
                for name, prm in m.named_parameters():
                    prm.copy_(P[f"{p}.{name}"])
            out[p] = m.eval().to(device=device, dtype=dtype)
    return out


def _lstm_module(P, p, x, lstms):
    """LSTMModule: 1x1 conv to one channel, nn.LSTM over frames, Linear + BatchNorm1d + ReLU -> [N, 1, nbins, nframes]"""
    N, _, nbins, nframes = x.shape
    h = _cbr_f(P, p + ".conv", x)[:, 0].permute(2, 0, 1)                     # [nframes, N, nbins]
    lstm = lstms[p + ".lstm"] if lstms is not None else lstm_modules({k: v for k, v in P.items() if k.startswith(p)})[p + ".lstm"]
    h, _ = lstm(h)
    h = F.linear(h.reshape(-1, h.shape[-1]), P[p + ".dense.0.weight"], P[p + ".dense.0.bias"])
    h = F.relu(_bn(P, p + ".dense.1", h))
    return h.reshape(nframes, N, 1, nbins).permute(1, 2, 3, 0)


def _up(x):
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)


def base_net(P, p, x, lstms=None):
    e = [_cbr_f(P, p + ".enc1", x)]
    for i in range(2, 6):
        e.append(_cbr_f(P, f"{p}.enc{i}.conv2", _cbr_f(P, f"{p}.enc{i}.conv1", e[-1], 2, "lrelu"), 1, "lrelu"))
    x = e[4]
    q = p + ".aspp"
    feats = [F.interpolate(_cbr_f(P, q + ".conv1.1", F.adaptive_avg_pool2d(x, (1, None))), size=x.shape[2:],
                           mode="bilinear", align_corners=True),
             _cbr_f(P, q + ".conv2", x)]
    feats += [_cbr_f(P, f"{q}.conv{i}", x, dil=d) for i, d in zip(range(3, 6), DILATIONS)]
    h = _cbr_f(P, q + ".bottleneck", torch.cat(feats, dim=1))
    for i in (4, 3, 2):
        h = _cbr_f(P, f"{p}.dec{i}.conv1", torch.cat([_up(h), e[i - 1]], dim=1))
    h = torch.cat([h, _lstm_module(P, p + ".lstm_dec2", h, lstms)], dim=1)
    return _cbr_f(P, p + ".dec1.conv1", torch.cat([_up(h), e[0]], dim=1))


def forward(P, x_mag, n_fft=1344, lstms=None):
    """CascadedNet(n_fft).forward in eval mode: the mask [B, 2, n_fft // 2 + 1, W]"""
    max_bin, out_bin = n_fft // 2, n_fft // 2 + 1
    x = x_mag[:, :, :max_bin]
    bw = max_bin // 2
    l1_in, h1_in = x[:, :, :bw], x[:, :, bw:]
    l1 = _cbr_f(P, "stg1_low_band_net.1", base_net(P, "stg1_low_band_net.0", l1_in, lstms))
    h1 = base_net(P, "stg1_high_band_net", h1_in, lstms)
    aux1 = torch.cat([l1, h1], dim=2)
    l2 = _cbr_f(P, "stg2_low_band_net.1", base_net(P, "stg2_low_band_net.0", torch.cat([l1_in, l1], dim=1), lstms))
    h2 = base_net(P, "stg2_high_band_net", torch.cat([h1_in, h1], dim=1), lstms)
    aux2 = torch.cat([l2, h2], dim=2)
    f3 = base_net(P, "stg3_full_band_net", torch.cat([x, aux1, aux2], dim=1), lstms)
    mask = torch.sigmoid(F.conv2d(f3, P["out.weight"]))
    return F.pad(mask, (0, 0, 0, out_bin - mask.shape[2]), mode="replicate")


def predict(P, x_mag, aggressiveness=None, n_fft=1344, lstms=None):
    """CascadedNet(n_fft).predict in eval mode: x_mag [B, 2, n_fft // 2 + 1, W] -> (x * mask)[..., 64:-64]; aggressiveness
    is accepted and ignored, as in the reference."""
    return (x_mag * forward(P, x_mag, n_fft, lstms))[:, :, :, OFFSET:-OFFSET]


def inference(P, x_spec, aggressiveness, data, n_fft=1344):
    """SeparateVREcho.inference (SeparateVR's) on the CPU: complex x_spec [2, n_fft // 2 + 1, n_frame] ->
    (pred * coef, |x|, exp(1j angle(x)))."""
    x_mag = np.abs(x_spec)
    x_phase = np.angle(x_spec)
    coef = x_mag.max()
    x_pre = x_mag / coef
    n_frame = x_pre.shape[2]
    ws = data["window_size"]
    pad_l, pad_r, roi = make_padding(n_frame, ws, OFFSET)
    n_window = int(np.ceil(n_frame / roi))
    lstms = lstm_modules(P)

    def run(pad_l, pad_r, n_window):
        xp = np.pad(x_pre, ((0, 0), (0, 0), (pad_l, pad_r)), mode="constant")
        with torch.no_grad():
            out = [predict(P, torch.from_numpy(xp[None, :, :, i * roi: i * roi + ws]), aggressiveness, n_fft, lstms)[0].numpy()
                   for i in range(n_window)]
        return np.concatenate(out, axis=2)

    pred = run(pad_l, pad_r, n_window)[:, :, :n_frame]
    if data["tta"]:
        pred_tta = run(pad_l + roi // 2, pad_r + roi // 2, n_window + 1)[:, :, roi // 2:][:, :, :n_frame]
        return (pred + pred_tta) * 0.5 * coef, x_mag, np.exp(1.0j * x_phase)
    return pred * coef, x_mag, np.exp(1.0j * x_phase)
