"""GPU parity of best_fft / EvaluationDomain through the C ABI against the CPU oracle (bit-exact)."""
import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be, device_lists  # noqa: F401

pytestmark = pytest.mark.gpu


def _omega(orc, k):
    return orc.fr([pyref.omega(k)])[0]


@pytest.mark.parametrize("k", [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20])
def test_best_fft_matches_oracle(be, orc, k):
    a = orc.fr_random_chacha(1 << k, 0x5eed0001 + k)
    w = _omega(orc, k)
    got = be.best_fft(a, w, k)
    want = orc.best_fft(a, w, k)
    assert np.array_equal(got, want)


def test_best_fft_small_matches_python_dft(be, orc):
    """BASELINE config 1 shape (2^12 is covered above); here an O(n^2) big-int DFT, independent of the oracle."""
    k = 6
    vals = [pow(3, i, pyref.R_MOD) for i in range(1 << k)]
    got = orc.fr_ints(be.best_fft(orc.fr(vals), _omega(orc, k), k))
    assert got == pyref.dft(vals, pyref.omega(k))


@pytest.mark.parametrize("k", [21, 22, 23])
def test_best_fft_large_inverse_roundtrip_and_oracle(be, orc, k):
    """three-pass sizes: oracle equality plus the size-independent property ifft(fft(a)) == n*a."""
    a = orc.fr_random_chacha(1 << k, 0x5eed0100 + k)
    w = _omega(orc, k)
    got = be.best_fft(a, w, k)
    assert np.array_equal(got, orc.best_fft(a, w, k))
    winv = orc.fr([pow(pyref.omega(k), -1, pyref.R_MOD)])[0]
    # check a sample of ifft(fft(a)) against n * a
    idx = [0, 1, 2, (1 << k) - 1, 12345 % (1 << k), (1 << (k - 1))]
    ai = orc.fr_ints(a[idx]); bi = orc.fr_ints(be.best_fft(got, winv, k)[idx])
    assert bi == [(x << k) % pyref.R_MOD for x in ai]


def test_inverse_omega(be, orc):
    k = 12
    a = orc.fr_random_chacha(1 << k, 77)
    winv = orc.fr([pow(pyref.omega(k), -1, pyref.R_MOD)])[0]
    assert np.array_equal(be.best_fft(a, winv, k), orc.best_fft(a, winv, k))


@pytest.mark.parametrize("j,k", [(4, 4), (5, 8), (4, 12), (5, 13), (3, 10), (9, 11)])
def test_evaluation_domain_matches_oracle(be, orc, j, k):
    from spectre_b200.halo2 import EvaluationDomain
    d = EvaluationDomain(be, j, k)
    od = orc.Domain(j, k)
    assert d.extended_k == od.extended_k
    for name in ("omega", "omega_inv", "extended_omega", "extended_omega_inv", "g_coset", "g_coset_inv", "ifft_divisor", "extended_ifft_divisor"):
        assert np.array_equal(getattr(d, name), getattr(od, name)), name
    a = orc.fr_random_chacha(1 << k, 1000 + k)
    coeff = d.lagrange_to_coeff(a)
    assert np.array_equal(coeff, od.lagrange_to_coeff(a))
    assert np.array_equal(d.coeff_to_lagrange(coeff), a)
    ext = d.coeff_to_extended(coeff)
    assert np.array_equal(ext, od.coeff_to_extended(coeff))
    e = orc.fr_random_chacha(1 << d.extended_k, 2000 + k)
    assert np.array_equal(d.divide_by_vanishing_poly(e), od.divide_by_vanishing_poly(e))
    assert np.array_equal(d.extended_to_coeff(e), od.extended_to_coeff(e))
    # coset convention, independent of the oracle: ext[i] = p(zeta * w_ext^i)
    ci = orc.fr_ints(coeff[:8] if k >= 3 else coeff)
    if (1 << k) <= 16:
        full = orc.fr_ints(coeff)
        wext = orc.fr_ints(od.extended_omega)[0]
        for i in (0, 1, 5):
            x = pyref.ZETA * pow(wext, i, pyref.R_MOD) % pyref.R_MOD
            assert orc.fr_ints(ext[i])[0] == sum(c * pow(x, e_, pyref.R_MOD) for e_, c in enumerate(full)) % pyref.R_MOD


@pytest.mark.parametrize("ids", device_lists(power_of_two=True))
def test_multi_device_six_step_ntt(orc, ids):
    """n_dev > 1 in one context: six-step NTT across devices (column blocks -> first pass -> one all-to-all over
    peer copies -> remaining passes -> strided gather). Must equal the oracle bit for bit, including the fused
    EvaluationDomain variants (zero padding / coset / truncation)."""
    from spectre_b200 import halo2
    be2 = halo2.Backend(ids)
    for k in (16, 17, 20, 22, 23):
        a = orc.fr_random_chacha(1 << k, 0x5eed0200 + k)
        w = _omega(orc, k)
        assert np.array_equal(be2.best_fft(a, w, k), orc.best_fft(a, w, k)), k
    j, k = 4, 16
    d = halo2.EvaluationDomain(be2, j, k)
    od = orc.Domain(j, k)
    a = orc.fr_random_chacha(1 << k, 99)
    coeff = d.lagrange_to_coeff(a)
    assert np.array_equal(coeff, od.lagrange_to_coeff(a))
    ext = d.coeff_to_extended(coeff)
    assert np.array_equal(ext, od.coeff_to_extended(coeff))
    e = orc.fr_random_chacha(1 << d.extended_k, 98)
    assert np.array_equal(d.extended_to_coeff(e), od.extended_to_coeff(e))
    be2.close()


@pytest.mark.parametrize("k", [24, 25])
def test_full_size_roundtrip_and_linearity(be, orc, k):
    """BASELINE extended-domain sizes (2^25 = K=23 extended): size-independent properties on device-resident data --
    ifft(fft(a)) == n*a (sampled), fft(a + b) == fft(a) + fft(b) (sampled), and fft of a delta is the all-ones / omega row."""
    import ctypes
    import torch
    n = 1 << k
    w = pyref.omega(k)
    omega = orc.fr([w])[0]; omega_inv = orc.fr([pow(w, -1, pyref.R_MOD)])[0]
    a = orc.fr_random_chacha(n, 0x5eed0300 + k)
    da = torch.from_numpy(a.view(np.int64)).cuda()
    orig = da.clone()
    be.best_fft_dev(da.data_ptr(), omega, k)
    fa = da.clone()
    be.best_fft_dev(da.data_ptr(), omega_inv, k)
    idx = [0, 1, 2, 3, n // 2, n - 1, 123457 % n, (1 << (k - 1)) + 5]
    back = orc.fr_ints(da[idx].cpu().numpy().view(np.uint64)); ai = orc.fr_ints(orig[idx].cpu().numpy().view(np.uint64))
    assert back == [(x << k) % pyref.R_MOD for x in ai]
    # X[0] = sum of inputs: check against a device-side reduction through eval_polynomial at x = 1
    s = orc.fr_ints(be.eval_polynomial_dev(orig.data_ptr(), n, orc.fr([1])[0]))[0]
    assert orc.fr_ints(fa[0:1].cpu().numpy().view(np.uint64))[0] == s
    # X[1] = p(omega)
    assert orc.fr_ints(fa[1:2].cpu().numpy().view(np.uint64))[0] == orc.fr_ints(be.eval_polynomial_dev(orig.data_ptr(), n, omega))[0]
    # delta at position 1 -> row of powers of omega
    d = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    d[1] = torch.from_numpy(orc.fr([1])[0].view(np.int64)).cuda()
    be.best_fft_dev(d.data_ptr(), omega, k)
    got = orc.fr_ints(d[idx].cpu().numpy().view(np.uint64))
    assert got == [pow(w, i, pyref.R_MOD) for i in idx]
