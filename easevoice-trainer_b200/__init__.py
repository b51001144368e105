"""easevoice-trainer_b200: H100-native (sm_90a) implementation of EaseVoice Trainer's stage-2 hot path.

Host code is Python (as the reference is); every kernel is hand-written CUDA behind the C ABI in
``include/evk.h`` (``libevk_sm90.so``).  There is no CPU fallback: ops raise if the library or an
H100 is missing.
"""
__version__ = "0.1.0"
