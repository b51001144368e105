"""Weights of the inference models that load a reference state_dict into host dicts: the one strict check of such a
state_dict, and moving the host dicts to a device."""
import torch


def _few(keys):
    return f"{keys[:5]}{'...' if len(keys) > 5 else ''}"


def check_state_dict(sd, spec, what):
    """Raise ValueError unless sd holds exactly the keys of spec ({key: shape}), each a floating-point tensor (fp16, fp32,
    ...) of its shape.  what names the model in the message."""
    missing = [k for k in spec if k not in sd]
    unexpected = [k for k in sd if k not in spec]
    if missing or unexpected:
        raise ValueError(f"state_dict does not match {what}: missing {_few(missing)}, unexpected {_few(unexpected)}")
    for k, shape in spec.items():
        v = sd[k]
        if not torch.is_tensor(v) or not v.is_floating_point() or tuple(v.shape) != tuple(shape):
            raise ValueError(f"{what}: {k}: expected a float tensor of shape {tuple(shape)}, got "
                             f"{f'{v.dtype} {tuple(v.shape)}' if torch.is_tensor(v) else type(v).__name__}")


def to_device(tree, device):
    """A dict of tensors, or a dict of such dicts, with every tensor moved to device; other values are kept as they are."""
    out = {}
    for k, v in tree.items():
        if isinstance(v, dict):
            v = to_device(v, device)
        elif torch.is_tensor(v):
            v = v.to(device)
        out[k] = v
    return out
