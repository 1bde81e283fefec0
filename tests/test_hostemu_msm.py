"""CPU-only test of the MSM pipeline (spectre_b200/csrc/msm.cuh): the per-thread bodies the CUDA kernels call are
run serially by tests/hostemu and compared with the oracle's best_multiexp and with Python big-int EC math."""
import ctypes

import numpy as np
import pytest

from tests import pyref
from tests.test_hostemu import _build, _p


@pytest.fixture(scope="module")
def he():
    return _build("libhostemu_ptx.so", ["-DSPB_EMULATE_PTX"])


def he_msm(he, scalars, bases, c=0, L=0, cap=24, precomp=0):
    scalars = np.ascontiguousarray(scalars, dtype=np.uint64); bases = np.ascontiguousarray(bases, dtype=np.uint64)
    out = np.empty(8, dtype=np.uint64)
    giants = ctypes.c_uint32(0)
    he.he_msm.restype = ctypes.c_uint64
    M = he.he_msm(_p(out), _p(scalars), _p(bases), ctypes.c_size_t(scalars.shape[0]), ctypes.c_uint32(c), ctypes.c_uint32(L), ctypes.c_uint32(cap), ctypes.byref(giants), ctypes.c_int(precomp))
    return out, int(M), giants.value


def oracle_affine(orc, scalars, bases):
    return orc.g1_to_affine(orc.best_multiexp(scalars, bases, threads=8))


@pytest.fixture(scope="module")
def points(orc):
    sc = orc.fr_random_chacha(600, 0x5eed0002)
    return orc.g1_fixed_base_mul(sc)


@pytest.mark.parametrize("n,c,L", [(1, 0, 0), (2, 3, 2), (7, 4, 3), (33, 5, 4), (100, 8, 32), (257, 7, 5), (600, 10, 32), (600, 0, 0), (600, 16, 32), (64, 20, 8),
                                   (300, 19, 32)])
def test_uniform_scalars(he, orc, points, n, c, L):
    sc = orc.fr_random_chacha(n, 0x5eed0003 + n)
    want = oracle_affine(orc, sc, points[:n])
    got, M, _ = he_msm(he, sc, points[:n], c, L)
    assert np.array_equal(got, want)
    # precomputed 2^(c*j) tables, single bucket set; c = 19 is the only width whose bucket reduction has more row blocks
    # than column blocks (nbr = 2, nbc = 1 in msm_tail_shape), so msm_tail_finish folds the two kinds over different counts
    if c <= 12 or c == 19:
        got, M, _ = he_msm(he, sc, points[:n], c, L, precomp=1)
        assert np.array_equal(got, want)


def test_against_python_ec(he, orc, points):
    n = 12
    ks = [3, 0, 1, pyref.R_MOD - 1, 2**128 + 5, 7, 2**253 + 11, 1, 1, 65535, 65536, 32768]
    sc = orc.fr(ks)
    got, _, _ = he_msm(he, sc, points[:n], 6, 4)
    pts = [pyref.aff_tuple(t) for t in orc.affine_ints(points[:n])]
    assert pyref.aff_tuple(orc.affine_ints(got)[0]) == pyref.msm(ks, pts)


@pytest.mark.parametrize("label", ["all_zero", "all_one", "all_minus_one", "single_nonzero", "dup_bases", "identity_bases", "cancel", "witness_like"])
def test_edge_distributions(he, orc, points, label):
    n = 300
    bases = points[:n].copy()
    rng = np.random.default_rng(5)
    if label == "all_zero":
        ks = [0] * n
    elif label == "all_one":
        ks = [1] * n
    elif label == "all_minus_one":
        ks = [pyref.R_MOD - 1] * n
    elif label == "single_nonzero":
        ks = [0] * n; ks[123] = 0xdeadbeefcafebabe1234567
    elif label == "dup_bases":
        ks = [int(x) for x in rng.integers(1, 1 << 62, n)]
        bases[:] = bases[0]                      # every bucket sees P + P: exercises the doubling branch
    elif label == "identity_bases":
        ks = [int(x) for x in rng.integers(1, 1 << 62, n)]
        bases[::3] = 0                           # halo2's (0,0) identity as a base
    elif label == "cancel":
        ks = [5] * n
        half = n // 2
        bases[half:2 * half] = bases[:half]
        bases[half:2 * half, 4:] = orc.fq([(-y) % pyref.P_MOD for y in orc.fq_ints(bases[:half, 4:])])  # P and -P in one bucket
    else:  # witness-like: 70% zero, 20% < 2^16, 9% < 2^104, 1% uniform (SURVEY.md 8d)
        ks = []
        for i in range(n):
            u = rng.random()
            ks.append(0 if u < 0.7 else int(rng.integers(0, 1 << 16)) if u < 0.9 else int(rng.integers(0, 1 << 62)) ** 2 % (1 << 104) if u < 0.99 else int(rng.integers(1, 1 << 62)) ** 4 % pyref.R_MOD)
    sc = orc.fr(ks)
    want = oracle_affine(orc, sc, bases)
    for c, L, cap, pre in ((0, 0, 24, 0), (4, 3, 2, 0), (9, 8, 1, 0), (6, 5, 3, 1), (0, 0, 24, 1), (19, 32, 24, 0), (19, 32, 24, 1)):
        got, M, giants = he_msm(he, sc, bases, c, L, cap, pre)
        assert np.array_equal(got, want), (label, c, L, pre)
    if label == "all_zero":
        assert M == 0 and not got.any()
    if label == "all_one":
        # one giant bucket: chains longer than the cap must have taken the block path
        got, M, giants = he_msm(he, sc, bases, 8, 4, 3)
        assert giants >= 1 and np.array_equal(got, want)


def test_geometry_choice(he):
    c = ctypes.c_uint32(); W = ctypes.c_uint32()
    for n, pre, lo, hi in ((1, 0, 3, 8), (1 << 10, 0, 6, 12), (1 << 20, 0, 15, 17), (1 << 23, 0, 16, 20), (1 << 24, 0, 17, 20),
                           (1 << 20, 1, 19, 21), (1 << 23, 1, 21, 22)):
        he.he_geometry(ctypes.c_uint64(n), ctypes.c_int(pre), ctypes.byref(c), ctypes.byref(W))
        # W*c >= 255 keeps one spare bit above the 254-bit scalar so the signed-digit carry never leaves the top window
        assert lo <= c.value <= hi and W.value * c.value >= 255 and (W.value - 1) * c.value < 255


def test_g_to_lagrange_of_the_seed0_srs(he, orc):
    """ParamsKZG::downsize recomputes g_lagrange = g_to_lagrange(g) (inverse DFT over the group). For the seed-0 SRS that must
    reproduce the Lagrange basis the oracle derives from the known secret -- the derivation the verifier contracts pin."""
    from tests import pyref
    for k in (0, 1, 3, 5):
        n = 1 << k
        g = orc.srs_g(k, 0, n)
        w = pow(pow(7, (pyref.R_MOD - 1) >> 28, pyref.R_MOD), 1 << (28 - k), pyref.R_MOD)
        w_inv = orc.fr([pow(w, -1, pyref.R_MOD)]); n_inv = orc.fr([pow(n, -1, pyref.R_MOD)])
        out = np.empty((n, 8), dtype=np.uint64)
        he.he_g_to_lagrange(_p(out), _p(np.ascontiguousarray(g)), ctypes.c_uint32(k), _p(w_inv), _p(n_inv))
        assert np.array_equal(out, orc.srs_g_lagrange(k, 0, n)), k


def test_long_chunks_are_chosen_from_the_real_entry_count(orc, points):
    """msm_effective_chunk (msm.cuh): the host asks for the long chunk (96 entries) from the upper bound n * W, the kernels use it
    only when the sorted list really has that many entries and fall back to 32 otherwise -- accumulate, stitch and the giant
    path must agree on the same effective length. Built with the threshold lowered to 2000 entries: a uniform column (about
    6000 entries: long chunks), a witness-like one (most digits dropped: short chunks) and a column of equal scalars (one
    chain across every chunk) all give the oracle's point."""
    he = _build("libhostemu_ptx_longchunk.so", ["-DSPB_EMULATE_PTX", "-DSPB_LONG_CHUNK_MIN_ENTRIES=2000"])
    n = 600
    rng = np.random.default_rng(3)
    uniform = orc.fr_random_chacha(n, 0xc4)
    sparse = orc.fr([0 if rng.random() < 0.8 else int(rng.integers(1, 1 << 16)) for _ in range(n)])
    equal = orc.fr([12345] * n)
    for sc, lo, hi in ((uniform, 2000, 1 << 30), (sparse, 1, 1999), (equal, 1, 1 << 30)):
        want = oracle_affine(orc, sc, points[:n])
        for precomp in (0, 1):
            got, M, _ = he_msm(he, sc, points[:n], c=10, L=96, precomp=precomp)
            assert np.array_equal(got, want)
            assert lo <= M <= hi, M
