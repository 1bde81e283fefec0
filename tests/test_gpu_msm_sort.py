"""The MSM's digit sort on the GPU (spectre_b200/csrc/msm.cuh steps 1-3: digit kernel, radix sort of the M entries by key,
bucket offsets) at the shapes where it branches, against the O(n) known-secret commitment of the seed-0 SRS
(orc.commit_known_tau, which uses no MSM code).

- Key widths: the sort looks at the bit length of the largest bucket key BW * B - 1 only, which CUB's onesweep radix sort
  covers in passes of 8 bits: 8 bits (one pass; lists that short take CUB's single-tile sort), 12 and 14 bits (two), 17
  and 19 bits (three), with and without window tables.
- M = 0 (the sort and the offsets kernel on an empty list) and M on both sides of kLongChunkMinEntries, where the kernels
  after the sort switch chunk length; spb_last_msm_adds = M + 2 * BW * B pins M.
- A context that lists device 0 twice: every part's digit kernel is queued before the host reads the first entry count.
- A batch whose lanes alternate sparse and dense columns, so every lane sorts lists of very different lengths in turn."""
import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be  # noqa: F401

pytestmark = pytest.mark.gpu

R = pyref.R_MOD
LONG_CHUNK_MIN_ENTRIES = 1 << 23   # msm.cuh kLongChunkMinEntries


def _mont(be, orc, canon):
    """canonical limbs (n, 4), each value below r -> Montgomery limbs, by one device product with R^2 mod r"""
    return be.vec_scale(canon, orc.fr([(1 << 256) % R])[0])


def _digit_column(be, orc, rng, c, counts):
    """scalar i = sum_{w < counts[i]} d_w 2^(c w) with 1 <= d_w <= B = 2^(c-1): exactly counts[i] non-zero signed digits,
    no carries, so the column has M = sum(counts) entries"""
    n = len(counts)
    canon = np.zeros((n, 4), dtype=np.uint64)
    for w in range(int(counts.max())):
        d = rng.integers(1, (1 << (c - 1)) + 1, n, dtype=np.uint64) * (counts > w).astype(np.uint64)
        limb, sh = divmod(c * w, 64)
        canon[:, limb] |= d << np.uint64(sh)
        if sh + c > 64:
            canon[:, limb + 1] |= d >> np.uint64(64 - sh)
    assert c * int(counts.max()) < 253
    return _mont(be, orc, canon)


def _witness(be, orc, n, rng):
    """70 % zero, 20 % below 2^16, 9 % below 2^104, 1 % uniform"""
    u = rng.random(n)
    canon = np.zeros((n, 4), dtype=np.uint64)
    small, mid = (u >= 0.7) & (u < 0.9), (u >= 0.9) & (u < 0.99)
    canon[small, 0] = rng.integers(0, 1 << 16, int(small.sum()), dtype=np.uint64)
    canon[mid, 0] = rng.integers(0, 1 << 63, int(mid.sum()), dtype=np.uint64)
    canon[mid, 1] = rng.integers(0, 1 << 40, int(mid.sum()), dtype=np.uint64)
    col = _mont(be, orc, canon)
    big = np.nonzero(u >= 0.99)[0]
    col[big] = orc.fr_random_chacha(len(big), 0x50f7)
    return col


def _same(orc, got, col):
    return np.array_equal(orc.g1_to_affine(got), orc.commit_known_tau(col))


def _buckets(be, n, tables):
    c, W = be.msm_geometry(n, tables)
    return c, (1 if tables else W) << (c - 1)


@pytest.fixture(scope="module")
def srs20(be, orc):
    """the seed-0 SRS of 2^20 points with window tables (c = 20, one bucket set of 2^19: 19-bit keys)"""
    from spectre_b200.halo2 import ParamsKZG
    p = ParamsKZG.setup(be, 20, orc.srs_tau()).precompute()
    yield p
    del p
    be.release_workspace()


@pytest.mark.parametrize("k,tables,key_bits", [(7, True, 8), (10, False, 12), (14, True, 14), (16, False, 17)])
def test_key_widths(be, orc, k, tables, key_bits):
    from spectre_b200.halo2 import ParamsKZG
    n = 1 << k
    c, nb = _buckets(be, n, tables)
    assert (nb - 1).bit_length() == key_bits
    p = ParamsKZG.setup(be, k, orc.srs_tau())
    if tables:
        p.precompute()
    rng = np.random.default_rng(k)
    for name, col in (("uniform", orc.fr_random_chacha(n, 0x5047 + k)), ("witness", _witness(be, orc, n, rng)),
                      ("ones", np.repeat(orc.fr([1]), n, axis=0))):
        assert _same(orc, p.commit(col), col), "%d-bit keys, %s column" % (key_bits, name)
    assert be.last_msm_adds == n + 2 * nb    # the column of ones: one entry per scalar
    del p


def test_three_pass_keys_and_empty_list(be, orc, srs20):
    n = 1 << 20
    c, nb = _buckets(be, n, True)
    assert (nb - 1).bit_length() == 19
    col = orc.fr_random_chacha(n, 0x5048)
    assert _same(orc, srs20.commit(col), col)
    for m in (n, 1000, 1):   # M = 0 over the whole basis and over short prefixes
        zero = np.zeros((m, 4), dtype=np.uint64)
        assert _same(orc, srs20.commit(zero), zero)
        assert be.last_msm_adds == 2 * nb
    zero = np.zeros((1 << 14, 4), dtype=np.uint64)     # and without tables: spb_msm_raw, one bucket set per window
    assert _same(orc, be.best_multiexp(zero, srs20.get_g(0, 1 << 14)), zero)
    assert be.last_msm_adds == 2 * _buckets(be, 1 << 14, False)[1]


@pytest.mark.parametrize("M", [LONG_CHUNK_MIN_ENTRIES - 1, LONG_CHUNK_MIN_ENTRIES, LONG_CHUNK_MIN_ENTRIES + 1])
def test_entry_count_across_the_long_chunk_threshold(be, orc, srs20, M):
    """2^20 scalars of 8 digits each make exactly 2^23 entries; one scalar with one digit fewer or more moves M across"""
    n = 1 << 20
    c, nb = _buckets(be, n, True)
    counts = np.full(n, 8, dtype=np.int64)
    counts[12345] += M - LONG_CHUNK_MIN_ENTRIES
    col = _digit_column(be, orc, np.random.default_rng(M), c, counts)
    assert _same(orc, srs20.commit(col), col)
    assert be.last_msm_adds == M + 2 * nb


@pytest.mark.parametrize("tables", [False, True])
def test_sharded_over_an_aliased_device_list(orc, tables):
    from spectre_b200 import halo2
    b2 = halo2.Backend([0, 0])
    try:
        k = 16
        n = 1 << k
        p = halo2.ParamsKZG.setup(b2, k, orc.srs_tau())
        if tables:
            p.precompute()
        rng = np.random.default_rng(16 + tables)
        cols = [("uniform", orc.fr_random_chacha(n, 0x5049)), ("witness", _witness(b2, orc, n, rng)), ("zero", np.zeros((n, 4), dtype=np.uint64)),
                ("first half zero", np.concatenate([np.zeros((n // 2, 4), dtype=np.uint64), orc.fr_random_chacha(n // 2, 0x504a)]))]
        for name, col in cols:
            assert _same(orc, p.commit(col), col), "[0, 0] %s" % name
        got = p.commit_batch(halo2.BASIS_G, [c for _, c in cols])
        for (name, col), g in zip(cols, got):
            assert _same(orc, g, col), "[0, 0] batch %s" % name
        del p
    finally:
        b2.close()


def test_batch_mixes_sparse_and_dense_columns(be, orc, srs20):
    from spectre_b200 import halo2
    n = 1 << 20
    c, _ = _buckets(be, n, True)
    rng = np.random.default_rng(20)
    ones = np.zeros(n, dtype=np.int64)
    ones[rng.integers(0, n, 300)] = 1
    cols = [("uniform", orc.fr_random_chacha(n, 0x504b)), ("zero", np.zeros((n, 4), dtype=np.uint64)), ("witness", _witness(be, orc, n, rng)),
            ("300 single digits", _digit_column(be, orc, rng, c, ones)), ("uniform", orc.fr_random_chacha(n, 0x504c)),
            ("all r - 1", np.repeat(orc.fr([R - 1]), n, axis=0)), ("witness", _witness(be, orc, n, rng)), ("zero", np.zeros((n, 4), dtype=np.uint64))]
    got = srs20.commit_batch(halo2.BASIS_G, [col for _, col in cols])
    bad = [name for (name, col), g in zip(cols, got) if not _same(orc, g, col)]
    assert not bad, bad
