"""Statistical quality of the attention probability-dropout draw (csrc/flash.cu: drop_row / drop_pair / drop_one), restated
here in numpy uint32 arithmetic.  The draw was made as cheap as a counter-based generator can be (one multiply-compare per element:
the attention kernels are bound by the integer pipe), so its statistics are checked explicitly: drop fraction, per-row / per-column
fractions at the binomial spread, no correlation between neighbouring columns, the two draws of a column pair, rows, diagonals."""
import numpy as np
import pytest

M32 = np.uint64(0xFFFFFFFF)
C, M1, M2 = 0xC2B2AE3D, 0x7FEB352D, 0x846CA68B         # DROP_C, DROP_M1, DROP_M2


def _u32(x):
    return (x & M32).astype(np.uint64)


def drop_row(row, s0):
    x = _u32(row * np.uint64(0x9E3779B1) + np.uint64(s0))
    x ^= x >> np.uint64(15); x = _u32(x * np.uint64(0x85EBCA77)); x ^= x >> np.uint64(13); x = _u32(x * np.uint64(0xC2B2AE35)); x ^= x >> np.uint64(16)
    return x


def keep_matrix(z, L, s0, s1, p):
    thr = np.uint64(min(max(p * 4294967296.0, 1.0), 4294967295.0))
    rh = drop_row(np.arange(L, dtype=np.uint64) + np.uint64(z * L), s0)[:, None]
    cols = np.arange(L, dtype=np.uint64)
    h = rh ^ _u32((cols >> np.uint64(1)) * np.uint64(C) + np.uint64(s1))[None, :]
    x = np.where((cols & np.uint64(1)).astype(bool)[None, :], _u32(h * np.uint64(M2)), _u32(h * np.uint64(M1)))
    return x >= thr


def _corr(a, b):
    a = a - a.mean(); b = b - b.mean()
    return float((a * b).mean() / np.sqrt((a * a).mean() * (b * b).mean()))


@pytest.mark.parametrize("p", [0.1, 0.25])
def test_dropout_draw_statistics(p):
    rng = np.random.default_rng(7)
    L = 1024
    for z in range(3):
        s0, s1 = int(rng.integers(0, 2 ** 32)), int(rng.integers(0, 2 ** 32))
        d = 1.0 - keep_matrix(z, L, s0, s1, p).astype(np.float64)
        n = d.size
        assert abs(d.mean() - p) < 4 * np.sqrt(p * (1 - p) / n) + 1e-4, d.mean()
        binom = np.sqrt(p * (1 - p) / L)
        assert 0.85 * binom < d.mean(1).std() < 1.15 * binom and 0.85 * binom < d.mean(0).std() < 1.15 * binom
        lim = 5.0 / np.sqrt(n)                                    # ~5 sigma of a sample correlation of independent draws
        for name, c in (("col+1", _corr(d[:, :-1], d[:, 1:])), ("pair", _corr(d[:, 0::2], d[:, 1::2])), ("col+2", _corr(d[:, :-2], d[:, 2:])),
                        ("row+1", _corr(d[:-1], d[1:])), ("diag", _corr(d[:-1, :-1], d[1:, 1:])), ("row+2", _corr(d[:-2], d[2:]))):
            assert abs(c) < lim, (name, c, lim)


def test_dropout_draw_differs_between_heads_and_streams():
    a = keep_matrix(0, 256, 123, 456, 0.1)
    assert (a != keep_matrix(1, 256, 123, 456, 0.1)).mean() > 0.1          # another (batch, head): rows hash differently
    assert (a != keep_matrix(0, 256, 124, 456, 0.1)).mean() > 0.1          # another seed word
    assert (a != keep_matrix(0, 256, 123, 457, 0.1)).mean() > 0.1
