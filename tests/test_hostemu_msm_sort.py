"""CPU-only test of the MSM's digit sort (spectre_b200/csrc/msm.cuh, steps 1-3): the digit and offsets bodies of the
library's kernels around a serial stable sort, against the counting sort (msm_count_thread / msm_scatter_thread and an
exclusive scan) on the same scalars.

tests/hostemu/msm_sort.cpp is compiled for the host with -DSPB_EMULATE_PTX (the Montgomery conversion as the GPU runs it)
and without it. Both sorts must give the same entry count M, the same bucket offsets (every bucket, empty ones included,
and offsets[BW * B] = M) and the same multiset of (key, index | sign) entries in every bucket; order inside a bucket may
differ. Keys stay below 2^key_bits, the bit range the device's radix sort looks at. The columns: uniform, all zero, all
r - 1 (one bucket per window), witness-like (mostly zero and small values) and single-digit (one non-zero digit per
scalar), in both geometries: one bucket set per window, and one set for all windows (window tables)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import pyref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu")
R = pyref.R_MOD
M64 = (1 << 64) - 1
N = 3000


@pytest.fixture(scope="module", params=["ptx", "native"])
def he(request, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostemu_msm_sort") / ("libhostemu_%s.so" % request.param))
    flags = ["-DSPB_EMULATE_PTX"] if request.param == "ptx" else []
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, os.path.join(HERE, "msm_sort.cpp")])
    lib = ctypes.CDLL(so)
    for f in ("he_sort_counting", "he_sort_radix", "he_sort_buckets"):
        getattr(lib, f).restype = ctypes.c_uint64
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _mont(vals):
    """canonical integers below r -> (n, 4) Montgomery limbs"""
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        m = (v << 256) % R
        out[i] = [(m >> (64 * j)) & M64 for j in range(4)]
    return out


def _column(name, c, rng):
    W = (255 + c - 1) // c
    if name == "uniform":
        return [int.from_bytes(rng.bytes(32), "little") % R for _ in range(N)]
    if name == "zero":
        return [0] * N
    if name == "minus_one":
        return [R - 1] * N
    if name == "witness":
        out = []
        for u in rng.random(N):
            if u < 0.7:
                out.append(0)
            elif u < 0.9:
                out.append(int(rng.integers(0, 1 << 16)))
            elif u < 0.99:
                out.append(int(rng.integers(0, 1 << 52)) << 52 | int(rng.integers(0, 1 << 52)))
            else:
                out.append(int.from_bytes(rng.bytes(32), "little") % R)
        return out
    if name == "single_digit":
        # d * 2^(c w) with 1 <= d <= B = 2^(c-1): one digit, no carry; windows kept below r
        B, out = 1 << (c - 1), []
        for _ in range(N):
            while True:
                v = int(rng.integers(1, B + 1)) << (c * int(rng.integers(0, W)))
                if v < R:
                    break
            out.append(v)
        return out
    raise KeyError(name)


def _sorted_by_bucket(ent, M):
    """(key, val) pairs sorted by key then val: equal for two lists iff every bucket holds the same multiset"""
    e = ent[:M]
    order = np.lexsort((e[:, 1], e[:, 0]))
    return e[order]


@pytest.mark.parametrize("precomp,c", [(0, 4), (0, 9), (0, 13), (1, 7), (1, 10), (1, 16)])
@pytest.mark.parametrize("name", ["uniform", "zero", "minus_one", "witness", "single_digit"])
def test_radix_sort_matches_counting_sort(he, name, precomp, c):
    rng = np.random.default_rng(1000 * c + 7 * precomp + len(name))
    vals = _column(name, c, rng)
    sc = _mont(vals)
    W = (255 + c - 1) // c
    nb = int(he.he_sort_buckets(ctypes.c_uint32(c), ctypes.c_int(precomp)))
    key_bits = he.he_sort_key_bits(ctypes.c_uint32(c), ctypes.c_int(precomp))
    assert nb == (1 if precomp else W) << (c - 1) and key_bits == (nb - 1).bit_length()
    got = {}
    for f in ("he_sort_counting", "he_sort_radix"):
        offsets = np.zeros(nb + 1, dtype=np.uint32)
        ent = np.zeros((N * W + 1, 2), dtype=np.uint32)
        M = int(getattr(he, f)(_p(sc), ctypes.c_uint64(N), ctypes.c_uint32(c), ctypes.c_int(precomp), _p(offsets), _p(ent)))
        keys = ent[:M, 0]
        assert np.all(keys[1:] >= keys[:-1]), f + ": entries not sorted by key"
        assert M == 0 or int(keys[-1]) < (1 << key_bits)
        got[f] = (M, offsets, _sorted_by_bucket(ent, M))
    (M0, off0, e0), (M1, off1, e1) = got["he_sort_counting"], got["he_sort_radix"]
    assert M1 == M0 and off1[nb] == M1
    assert np.array_equal(off1, off0), "bucket offsets differ"
    assert np.array_equal(e1, e0), "a bucket holds different entries"
    if name == "zero":
        assert M1 == 0
    if name == "single_digit":
        assert M1 == N
    if name == "minus_one":
        assert np.count_nonzero(np.diff(off1)) == len(set(e1[:, 0].tolist()))   # one bucket per window with a non-zero digit
