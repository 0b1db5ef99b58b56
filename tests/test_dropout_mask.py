"""The host reference of the fused dropout mask (tests/dropout_ref.py): Philox4x32-10 itself, and the statistics of the
masks the kernels are compared against."""
import numpy as np
import pytest

from dropout_ref import dropout_mask, keep_threshold, philox4x32_10

# Random123 known-answer vectors of philox4x32_10: (counter, key) -> output
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("counter,key,expect", KAT)
def test_philox_known_answers(counter, key, expect):
    got = tuple(int(w) for w in philox4x32_10(counter, key))
    assert got == expect, [f"{w:08x}" for w in got]


def test_philox_is_elementwise():
    """the vectorised generator computes each element as the scalar one does"""
    rng = np.random.default_rng(0)
    c = rng.integers(0, 2 ** 32, (4, 50), dtype=np.uint64)
    key = (0x12345678, 0x9ABCDEF0)
    vec = philox4x32_10(tuple(c), key)
    for j in range(50):
        one = philox4x32_10(tuple(int(v) for v in c[:, j]), key)
        assert [int(w[j]) for w in vec] == [int(w) for w in one]


def test_keep_threshold_is_float32():
    assert int(keep_threshold(0.5)) == 2 ** 31
    assert int(keep_threshold(1.0)) == 4294967040              # clamped below 2^32
    assert int(keep_threshold(0.9)) == int(np.float32(0.9) * np.float32(2.0 ** 32))
    assert int(keep_threshold(0.9)) != int(0.9 * 2 ** 32)        # the float64 product would round differently


@pytest.mark.parametrize("keep", [0.3, 0.5, 0.75, 0.9])
def test_mask_statistics(keep):
    """kept fraction within 5 sigma of keep; masks at neighbouring counters, at two streams and at two seeds uncorrelated"""
    B, N = 600, 520                                              # 312000 elements; N is not a multiple of 4
    m = dropout_mask(B, N, keep, 0x1234567, 3, 10)
    n = m.size
    sigma = np.sqrt(keep * (1 - keep) / n)
    assert abs(m.mean() - keep) < 5 * sigma, (m.mean(), keep, sigma)
    # each of the four lanes of one Philox output, and the first / last rows and columns, on their own
    for lane in range(4):
        sub = m[:, lane::4]
        assert abs(sub.mean() - keep) < 5 * np.sqrt(keep * (1 - keep) / sub.size)
    others = {"counter + 1": dropout_mask(B, N, keep, 0x1234567, 3, 11),
              "another stream": dropout_mask(B, N, keep, 0x1234567, 4, 10),
              "another seed": dropout_mask(B, N, keep, 0x7654321, 3, 10)}
    for what, o in others.items():
        corr = np.corrcoef(m.ravel().astype(np.float64), o.ravel().astype(np.float64))[0, 1]
        assert abs(corr) < 0.01, f"keep {keep}: mask and the mask of {what} correlate ({corr:.3f})"
    # neighbouring elements of one row and one column are not correlated either
    x = m.astype(np.float64)
    for a, b in ((x[:, :-1], x[:, 1:]), (x[:-1], x[1:])):
        assert abs(np.corrcoef(a.ravel(), b.ravel())[0, 1]) < 0.01
