"""Launch accounting of the C ABI: zero-length calls launch nothing and leave no error behind, and every entry point reports
exactly the kernel launches it makes (spb_kernel_launches counts the library's own kernels, not CUB's, memsets or copies)."""
import ctypes

import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture
def fresh():
    """A backend of its own on device 0, so nothing earlier in the session has touched its counter or its workspace."""
    from spectre_b200 import halo2
    b = halo2.Backend([0])
    yield b
    b.close()


def _dev(a):
    """device copy of a host (n, 4) / (n, 8) uint64 array, complete before the library's (non-blocking) stream uses it"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def _vp(x):
    """ctypes pointer to a numpy array or a torch tensor's device memory"""
    return ctypes.c_void_p(x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data)


def _ptrs(*ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def test_zero_length_calls_launch_nothing(fresh, orc):
    """n = 0 (kate division: n = 1, an empty quotient) with valid pointers returns 0, launches nothing and leaves no CUDA error
    pending: a transform on the same thread afterwards succeeds and matches the oracle."""
    lib, ctx, Z = fresh.lib, fresh.ctx, ctypes.c_size_t(0)
    h, h2, s = orc.fr_random_chacha(1, 1), orc.fr_random_chacha(1, 2), orc.fr_random_chacha(1, 3)
    out_fr, out_g1 = np.zeros((1, 4), np.uint64), np.zeros((1, 8), np.uint64)
    d, d2, dout = _dev(h), _dev(h2), _dev(out_fr)
    calls = {
        "spb_vec_mul": lambda: lib.spb_vec_mul(ctx, _vp(h), _vp(h2), Z),
        "spb_vec_axpy": lambda: lib.spb_vec_axpy(ctx, _vp(h), _vp(s), _vp(h2), Z),
        "spb_vec_scale": lambda: lib.spb_vec_scale(ctx, _vp(h), _vp(s), Z),
        "spb_vec_mul_dev": lambda: lib.spb_vec_mul_dev(ctx, _vp(d), _vp(d2), Z),
        "spb_vec_axpy_dev": lambda: lib.spb_vec_axpy_dev(ctx, _vp(d), _vp(s), _vp(d2), Z),
        "spb_vec_scale_dev": lambda: lib.spb_vec_scale_dev(ctx, _vp(d), _vp(s), Z),
        "spb_lincomb_dev": lambda: lib.spb_lincomb_dev(ctx, _ptrs(d), ctypes.c_size_t(1), _vp(s), _vp(dout), Z),
        "spb_weighted_sum_dev": lambda: lib.spb_weighted_sum_dev(ctx, _ptrs(d), _vp(s), ctypes.c_size_t(1), _vp(dout), Z),
        "spb_g1_fixed_base_mul": lambda: lib.spb_g1_fixed_base_mul(ctx, _vp(s), Z, _vp(out_g1)),
        "spb_grand_product": lambda: lib.spb_grand_product(ctx, _vp(h), Z, _vp(out_fr)),
        "spb_grand_product_dev": lambda: lib.spb_grand_product_dev(ctx, _vp(d), Z, _vp(dout)),
        "spb_batch_invert": lambda: lib.spb_batch_invert(ctx, _vp(h), Z),
        "spb_batch_invert_dev": lambda: lib.spb_batch_invert_dev(ctx, _vp(d), Z),
        "spb_eval_polynomial": lambda: lib.spb_eval_polynomial(ctx, _vp(h), Z, _vp(s), _vp(out_fr)),
        "spb_eval_polynomial_dev": lambda: lib.spb_eval_polynomial_dev(ctx, _vp(d), Z, _vp(s), _vp(out_fr)),
        "spb_kate_division": lambda: lib.spb_kate_division(ctx, _vp(h), ctypes.c_size_t(1), _vp(s), _vp(out_fr)),
        "spb_kate_division_dev": lambda: lib.spb_kate_division_dev(ctx, _vp(d), ctypes.c_size_t(1), _vp(s), _vp(dout)),
    }
    for name, call in calls.items():
        before = fresh.kernel_launches
        rc = call()
        assert rc == 0, "%s with n = 0 returned %d: %s" % (name, rc, lib.spb_last_error(ctx).decode())
        assert fresh.kernel_launches == before, "%s with n = 0 launched a kernel" % name
    k = 10
    a = orc.fr_random_chacha(1 << k, 0x5eed0a00)
    w = orc.fr([pyref.omega(k)])[0]
    da = _dev(a)
    fresh.best_fft_dev(da.data_ptr(), w, k)
    assert np.array_equal(da.cpu().numpy().view(np.uint64), orc.best_fft(a, w, k))


def _counted(b, call):
    before = b.kernel_launches
    call()
    return b.kernel_launches - before


def _cases(b, orc):
    """{name: (expected launches, call)}; everything a call needs is made before it is counted"""
    from spectre_b200 import halo2
    n = 3001
    a, c, s = orc.fr_random_chacha(n, 10), orc.fr_random_chacha(n, 11), orc.fr_random_chacha(1, 12)[0]
    da, dc, dz = _dev(a), _dev(c), _dev(np.zeros((n, 4), np.uint64))
    lib, ctx = b.lib, b.ctx
    dom = halo2.EvaluationDomain(b, 4, 10)
    ext = orc.fr_random_chacha(dom.extended_len(), 13)
    dext = _dev(ext)
    params = halo2.ParamsKZG.setup(b, 8, orc.srs_tau())
    small = halo2.ParamsKZG.setup(b, 4, orc.srs_tau())
    k = 8
    cols = [_dev(orc.fr_random_chacha(1 << k, 20 + i)) for i in range(4)]
    dzk = _dev(np.zeros((1 << k, 4), np.uint64))
    blinds = orc.fr_random_chacha(3, 30)
    one = orc.fr([1])[0]

    def axpy_dev():
        b.check(lib.spb_vec_axpy_dev(ctx, _vp(da), _vp(s), _vp(dc), ctypes.c_size_t(n)), "spb_vec_axpy_dev")

    return {
        "spb_vec_mul": (1, lambda: b.vec_mul(a, c)),
        "spb_vec_axpy": (1, lambda: b.vec_axpy(a, s, c)),
        "spb_vec_scale": (1, lambda: b.vec_scale(a, s)),
        "spb_vec_mul_dev": (1, lambda: b.vec_mul_dev(da.data_ptr(), dc.data_ptr(), n)),
        "spb_vec_axpy_dev": (1, axpy_dev),
        "spb_vec_scale_dev": (1, lambda: b.vec_scale_dev(da.data_ptr(), s, n)),
        "spb_lincomb_dev": (1, lambda: b.lincomb_dev([da.data_ptr(), dc.data_ptr()], s, dz.data_ptr(), n)),
        "spb_weighted_sum_dev": (1, lambda: b.weighted_sum_dev([da.data_ptr(), dc.data_ptr()], [s, s], dz.data_ptr(), n)),
        "spb_eval_polynomial": (1, lambda: b.eval_polynomial(a, s)),
        "spb_eval_polynomial_dev": (1, lambda: b.eval_polynomial_dev(da.data_ptr(), n, s)),
        "spb_eval_polynomial_many_dev": (1, lambda: b.eval_polynomial_many_dev([da.data_ptr(), dc.data_ptr(), da.data_ptr()], n, [s, one, s])),
        "spb_fr_random_chacha_dev": (1, lambda: b.fr_random_chacha_dev(7, 0, dz.data_ptr(), n)),
        "spb_divide_by_vanishing": (1, lambda: dom.divide_by_vanishing_poly(ext)),
        "spb_divide_by_vanishing_dev": (1, lambda: dom.divide_by_vanishing_poly_dev(dext.data_ptr())),
        "spb_g1_fixed_base_mul": (1, lambda: b.g1_fixed_base_mul(a[:100])),
        "spb_domain_new": (1, lambda: halo2.EvaluationDomain(b, 3, 8)),
        "spb_product_dev": (2, lambda: b.product_dev(da.data_ptr(), n)),
        "spb_grand_product": (3, lambda: b.grand_product(a)),
        "spb_grand_product_dev": (3, lambda: b.grand_product_dev(da.data_ptr(), n, dz.data_ptr())),
        "spb_grand_product_seeded_dev": (3, lambda: b.grand_product_seeded_dev(da.data_ptr(), n, s, dz.data_ptr())),
        "spb_batch_invert": (3, lambda: b.batch_invert(a)),
        "spb_batch_invert_dev": (3, lambda: b.batch_invert_dev(da.data_ptr(), n)),
        "spb_kate_division": (3, lambda: b.kate_division(a, s)),
        "spb_kate_division_dev": (3, lambda: b.kate_division_dev(da.data_ptr(), n, s, dz.data_ptr())),
        "spb_permutation_product_dev": (8, lambda: b.permutation_product_dev(k, [t.data_ptr() for t in cols[:2]], [t.data_ptr() for t in cols[2:]], 0, s, s,
                                                                            blinds, one, dzk.data_ptr())),
        "spb_lookup_product_dev": (8, lambda: b.lookup_product_dev(1 << k, *[t.data_ptr() for t in cols], s, s, blinds, dzk.data_ptr())),
        "spb_msm_dev": (10, lambda: params.commit_dev(halo2.BASIS_G, da.data_ptr(), 1 << 8)),
        "spb_srs_downsize-k3": (3 + 3, lambda: small.downsize(3)),
        "spb_srs_downsize-k1": (3 + 1, lambda: small.downsize(1)),
        "spb_srs_downsize-k0": (2, lambda: small.downsize(0)),
    }


def test_launch_counts(fresh, orc):
    """Exact launches per entry point on a one-device context."""
    cases = _cases(fresh, orc)
    got = {name: _counted(fresh, call) for name, (_, call) in cases.items()}
    want = {name: expect for name, (expect, _) in cases.items()}
    assert got == want
