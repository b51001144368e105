"""Statistical quality of the attention probability-dropout draw (csrc/flash.cu: drop_row / drop_pair / drop_one), restated
in numpy uint32 arithmetic by tests/attention_ref.py.  The draw was made as cheap as a counter-based generator can be (one
multiply-compare per element: the attention kernels are bound by the integer pipe), so its statistics are checked explicitly:
drop fraction, per-row / per-column fractions at the binomial spread, no correlation between neighbouring columns, the two draws
of a column pair, rows, diagonals."""
import numpy as np
import pytest

from tests.attention_ref import keep_matrix, philox


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


def test_philox_known_answer():
    """Philox-4x32-10 test vectors of Random123 (Salmon et al., SC'11): key (k0, k1), counter (c0, c1, c2, c3)"""
    M = 0xFFFFFFFF
    assert philox(0, 0, 0) == (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    assert philox(M | M << 32, M | M << 32, M | M << 32) == (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)
