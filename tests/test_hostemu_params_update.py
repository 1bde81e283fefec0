"""CPU-only test of a powers-of-tau update's bodies (spb_srs_contribute): the per-point scale g'[j] = t^(start + j) g[j]
(spectre_b200/csrc/msm.cuh, srs_scale_thread) and the trailer's G2 multiple s_g2' = t s_g2 (spectre_b200/csrc/pairing.cuh,
g2_mul_scalar).

tests/hostemu/params_update.cpp is compiled for the host with -DSPB_EMULATE_PTX (the 32-bit-limb carry chains the GPU runs)
and without it. The scaled points of g[j] = s^j G1 must be the points of the secret s t, made by the oracle's fixed-base
multiplication as tests/test_params_check_cpu.secret_params makes them, at shard offsets 0 and past zero; the G2 multiple must
be tests/pypairing's g2_mul of the generator by s t. t runs over 1, 2, r - 1 and random values; the identity stays the identity."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from spectre_b200 import plonk
from tests import pypairing as pp

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu")
R = pp.R
N = 24


@pytest.fixture(scope="module", params=["ptx", "native"])
def he(request, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostemu_params_update") / ("libhostemu_%s.so" % request.param))
    flags = ["-DSPB_EMULATE_PTX"] if request.param == "ptx" else []
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, os.path.join(HERE, "params_update.cpp")])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _secrets():
    rng = random.Random(0x7a0)
    return [1, 2, R - 1] + [rng.randrange(2, R - 1) for _ in range(3)]


def _powers(orc, s, start, n):
    """s^(start + j) G1 for j < n, as (n, 8) affine limbs"""
    return orc.g1_fixed_base_mul(plonk.fr_mont_rows([pow(s, start + j, R) for j in range(n)]))


def scale(he, pts, start, t):
    pts = np.ascontiguousarray(pts, dtype=np.uint64)
    out = np.full(((pts.shape[0] + 1), 8), 0xA5A5, dtype=np.uint64)        # one row past the end: must stay as it is
    tm = plonk.fr_mont(t)
    he.he_srs_scale(_p(pts), _p(out), ctypes.c_uint64(start), ctypes.c_uint64(pts.shape[0]), _p(tm))
    assert (out[-1] == 0xA5A5).all()
    return out[:-1]


def g2_mul(he, q, t):
    q = np.ascontiguousarray(pp.g2_limbs(q))
    out = np.empty(16, dtype=np.uint64)
    tm = plonk.fr_mont(t)
    he.he_g2_mul(_p(q), _p(tm), _p(out))
    return pp.g2_from_limbs(out)


@pytest.mark.parametrize("start", [0, 1000])
def test_scaled_points_are_the_powers_of_s_t(he, orc, start):
    s = random.Random(start + 1).randrange(2, R)
    pts = _powers(orc, s, start, N)
    for t in _secrets():
        got = scale(he, pts, start, t)
        assert np.array_equal(got, _powers(orc, s * t % R, start, N)), t


def test_identity_points_stay_the_identity(he, orc):
    pts = _powers(orc, 5, 3, 8)
    pts[[0, 3, 7]] = 0
    for t in _secrets():
        got = scale(he, pts, 3, t)
        assert not got[[0, 3, 7]].any()
        want = _powers(orc, 5 * t % R, 3, 8)
        keep = [1, 2, 4, 5, 6]
        assert np.array_equal(got[keep], want[keep]), t


def test_g2_multiple_is_the_trailer_of_s_t(he):
    s = random.Random(9).randrange(2, R)
    q = pp.g2_mul(pp.G2_GEN, s)
    for t in _secrets():
        assert g2_mul(he, q, t) == pp.g2_mul(pp.G2_GEN, s * t % R), t
    assert g2_mul(he, q, R - 1) == pp.g2_neg(q)
    assert g2_mul(he, None, 12345) is None
    assert g2_mul(he, pp.G2_GEN, 0) is None
