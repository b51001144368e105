"""Float64 emulation of the UVR5 VR CascadedASPPNet, the DeEcho / DeReverb CascadedNet and MDX23C under a float16 /
bfloat16 compute type, as uvr5.py and mdx23c.py run them: both operands of every dense convolution rounded to nearest even
to 16 bits -- the input from its fp32 value, the conv weight as stored (unscaled: the BatchNorm after it stays in fp32) --
and everything else unrounded: BatchNorm scale and bias, the depthwise 3x3s, the bilinear resizes, the height mean, the
LSTM, the mask head, the instance norms, GELU, the TDF Linears, the transposed convs, the STFT and the iSTFT.

The emulation runs the oracles themselves (oracle/uvr5_oracle.py, uvr5_echo_oracle.py, mdx23c_oracle.py) in float64 on the
input's device, with their F.conv2d replaced by one that rounds the operands of a dense conv (groups == 1) other than the
mask head's.  With dtype None nothing is rounded, and the computation is the float64 restatement of the oracles."""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import mdx23c_oracle as MO
from oracle import uvr5_echo_oracle as EO
from oracle import uvr5_oracle as VO


def rounding(dtype):
    """-> h: x rounded to fp32, then to nearest even in `dtype`, as float64; the identity when dtype is None"""
    if dtype is None:
        return lambda x: x
    return lambda x: x.float().to(dtype).double()


class _RoundedConvF:
    """torch.nn.functional with conv2d rounding both operands of a dense conv whose weight is not one of `keep`"""

    def __init__(self, h, keep):
        self.h, self.keep = h, keep

    def __getattr__(self, name):
        return getattr(F, name)

    def conv2d(self, x, w, *args, **kw):
        groups = kw.get("groups", args[4] if len(args) > 4 else 1)
        if groups != 1 or any(w is k for k in self.keep):
            return F.conv2d(x, w, *args, **kw)
        return F.conv2d(self.h(x), self.h(w), *args, **kw)


@contextlib.contextmanager
def _rounded_convs(module, dtype, keep=()):
    """run `module`'s functions with the rounded conv2d of `dtype` (nothing changes for None)"""
    module.F = _RoundedConvF(rounding(dtype), keep)
    try:
        yield
    finally:
        module.F = F


def _double(P, device):
    return {k: (v.double().to(device) if v.is_floating_point() else v.to(device)) for k, v in P.items()}


@torch.no_grad()
def vr_predict(P, x_mag, aggressiveness, dtype, n_fft, enlarge):
    """CascadedASPPNet.predict of x_mag [B, 2, bins, W] (any float dtype, on any device) under `dtype` -> float64"""
    P = _double(P, x_mag.device)
    with _rounded_convs(VO, dtype, keep=(P["out.weight"],)):
        return VO.predict(P, x_mag.double(), aggressiveness, n_fft, enlarge)


@torch.no_grad()
def echo_predict(P, x_mag, dtype, n_fft, lstms=None):
    """CascadedNet.predict of x_mag [B, 2, bins, W] under `dtype` -> float64 (lstms: EO.lstm_modules(P) in float64 on
    x_mag's device, built once by the caller or here)"""
    P = _double(P, x_mag.device)
    if lstms is None:
        lstms = EO.lstm_modules(P, x_mag.device, torch.float64)
    with _rounded_convs(EO, dtype, keep=(P["out.weight"],)):
        return EO.predict(P, x_mag.double(), None, n_fft, lstms)


@torch.no_grad()
def inference(predict, x_spec, data, offset, device):
    """SeparateVR.inference (oracle/uvr5_oracle.py's window loop) with `predict` (windows [n, 2, bins, ws] float64 on device
    -> [n, 2, bins, ws - 2 offset]) in place of the net, every window in one call: -> pred * coef, float64 numpy.  The
    magnitudes are normalised in fp32, as uvr5.inference does before the copy to the device."""
    x_mag = np.abs(x_spec)
    x_pre = torch.from_numpy(np.ascontiguousarray(x_mag / x_mag.max(), dtype=np.float32)).double().to(device)
    n_frame, ws = x_pre.shape[2], data["window_size"]
    pad_l, pad_r, roi = VO.make_padding(n_frame, ws, offset)
    n_window = int(np.ceil(n_frame / roi))

    def run(pl, pr, n):
        xp = F.pad(x_pre, (pl, pr))
        wins = torch.stack([xp[:, :, i * roi:i * roi + ws] for i in range(n)])
        out = predict(wins)
        return torch.cat(list(out), 2).cpu().numpy()

    pred = run(pad_l, pad_r, n_window)[:, :, :n_frame]
    if data["tta"]:
        pred_tta = run(pad_l + roi // 2, pad_r + roi // 2, n_window + 1)[:, :, roi // 2:][:, :, :n_frame]
        pred = (pred + pred_tta) * 0.5
    return pred * float(x_mag.max())


@torch.no_grad()
def mdx_forward(P, cfg, raw, dtype):
    """TFC_TDF_net(cfg).forward(raw) under `dtype`, float64 on raw's device"""
    P = _double(P, raw.device)
    with _rounded_convs(MO, dtype):
        return MO.forward(P, cfg, raw.double())


def mdx_demix(P, cfg, mix, dtype, device):
    """SeparateMDXC.demix_track (oracle/mdx23c_oracle.py) with the emulated forward on `device`"""
    net = lambda chunks: mdx_forward(P, cfg, chunks.to(device), dtype).cpu()          # noqa: E731
    return MO.demix_track(net, mix.double(), cfg["audio"]["chunk_size"])
