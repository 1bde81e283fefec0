"""GPU: spb_permute_expression_pair_dev on the column shapes that reach each branch of its radix sort (skipped and
single-outlier digits, odd and even pass counts, stability across limbs and tiles), of its match (a value below, between
or above the table) and of its leftover hand-out (no repeated rows, n - 1 of them), from one row to 2^24 - 7; and
spb_lookup_product_dev past 2^20 rows, on the columns the device sort produced. Every result is bit-exact against the
oracle, matches the Python restatement up to 2^16 rows, and satisfies the lookup argument's definition."""
import numpy as np
import pytest

from tests.gpu_common import be  # noqa: F401
from tests.test_lookup_reference import (MISSING, PLACEMENTS, SHAPES, SMALL_SIZES, check_lookup_definition, make_shape, mont_pool,
                                         permute_reference, shape_missing, shape_spectre)

pytestmark = pytest.mark.gpu

PY_REFERENCE_MAX = 1 << 16


@pytest.fixture(scope="module", autouse=True)
def _free_module_buffers(be):
    """The 2^23- and 2^24-row columns grow the session context's lookup workspaces and torch's cached blocks by several GiB;
    give them back so that later modules can prove at K = 24 on the same device."""
    yield
    import torch
    torch.cuda.synchronize()
    be.release_workspace()
    torch.cuda.empty_cache()


def _dev(torch, arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _device_permute(be, torch, inp, tab):
    di, dt = _dev(torch, inp), _dev(torch, tab)
    oi, ot = torch.empty_like(di), torch.empty_like(dt)
    be.permute_expression_pair_dev(di.data_ptr(), dt.data_ptr(), inp.shape[0], oi.data_ptr(), ot.data_ptr())
    return oi, ot


def _check_permute(be, orc, pool, ii, ti):
    """device against the oracle (bit-exact), the Python restatement (up to 2^16 rows) and the definition"""
    import torch
    mp = mont_pool(orc, pool)
    inp, tab = mp[ii], mp[ti]
    oi, ot = _device_permute(be, torch, inp, tab)
    got_i, got_t = _host(oi), _host(ot)
    want_i, want_t = orc.permute_expression_pair(inp, tab)
    assert np.array_equal(got_i, want_i), "permuted input differs from the oracle"
    assert np.array_equal(got_t, want_t), "permuted table differs from the oracle"
    if inp.shape[0] <= PY_REFERENCE_MAX:
        p_in, p_tab = permute_reference([pool[int(i)] for i in ii], [pool[int(i)] for i in ti])
        assert orc.fr_ints(got_i) == p_in and orc.fr_ints(got_t) == p_tab
    check_lookup_definition(inp, tab, got_i, got_t)
    return inp, tab, oi, ot


@pytest.mark.parametrize("n", SMALL_SIZES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_permute_shape(be, orc, shape, n):
    _check_permute(be, orc, *make_shape(shape, n, seed=n))


@pytest.mark.parametrize("shape,n", [
    ("spectre", (1 << 16) - 7),       # K = 16, checked against the Python restatement too
    ("range12", 1 << 16),             # two passes on limb 0
    ("range19", (1 << 20) + 1),       # three passes on limb 0
    ("top_and_low", (1 << 20) + 3),   # stability across limbs and 513 tiles
    ("theta", (1 << 20) + 5),         # eight passes on every limb
    ("spectre", (1 << 20) - 7),       # K = 20
    ("range23", (1 << 23) - 7),       # three passes on limb 0 at the largest range-check size
    ("spectre", (1 << 23) - 7),       # K = 23
])
def test_permute_large(be, orc, shape, n):
    _check_permute(be, orc, *make_shape(shape, n, seed=n))


@pytest.mark.slow
def test_permute_committee_update_shape(be, orc):
    """K = 24: a 2^23 range table padded with zeros to 2^24 - 7 usable rows"""
    n = (1 << 24) - 7
    _check_permute(be, orc, *shape_spectre(23)(n, np.random.default_rng(24)))


@pytest.mark.parametrize("n", [2, 33, 2049])
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("where", MISSING)
def test_permute_missing_value(be, orc, where, placement, n):
    """a value missing from the table fails like upstream's Error::ConstraintSystemFailure; the next call on the same context,
    at another length, is unaffected by the failed one (scratch slots and the error flag are reset)"""
    import torch
    from spectre_b200.halo2 import BackendError
    pool, ii, ti = shape_missing(where, placement, n, seed=n)
    mp = mont_pool(orc, pool)
    with pytest.raises(BackendError, match="ConstraintSystemFailure"):
        _device_permute(be, torch, mp[ii], mp[ti])
    _check_permute(be, orc, *make_shape("spectre", 3 * n + 1, seed=n))


# ---- the lookup grand product ------------------------------------------------------------------------------------------
N_BLINDS = 6


def _lookup_product(be, orc, cols, beta, gamma, blinds):
    import torch
    n = cols[0].shape[0]
    d = [c if isinstance(c, torch.Tensor) else _dev(torch, c) for c in cols]
    dz = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    be.lookup_product_dev(n, *[t.data_ptr() for t in d], beta, gamma, blinds, dz.data_ptr())
    return _host(dz)


@pytest.mark.parametrize("zero_row", ["first", "last_usable"])
@pytest.mark.parametrize("n", [(1 << 16) + 3, (1 << 20) + 1, 1 << 22])
def test_lookup_product_zero_denominator(be, orc, n, zero_row):
    """a zero denominator stays zero through the batch inversion: on the first row it zeroes the rest of z, on the last
    usable row it must leave every other row's inverse alone"""
    cols = [orc.fr_random_chacha(n, 900 + i) for i in range(4)]
    beta, gamma = orc.fr_random_chacha(2, 910)
    if zero_row == "first":
        cols[2][0] = orc.fr([-orc.fr_ints(beta.reshape(1, 4))[0]])[0]              # permuted_input + beta = 0
    else:
        cols[3][n - N_BLINDS - 1] = orc.fr([-orc.fr_ints(gamma.reshape(1, 4))[0]])[0]   # permuted_table + gamma = 0
    blinds = orc.fr_random_chacha(N_BLINDS, 911).reshape(-1, 4)
    assert np.array_equal(_lookup_product(be, orc, cols, beta, gamma, blinds), orc.lookup_product(*cols, beta, gamma, blinds))


@pytest.mark.parametrize("k", [16, 20])
def test_lookup_product_of_device_sort(be, orc, k):
    """Spectre's lookup column at 2^k rows: the device sorts the 2^k - 7 usable rows, the blinding rows are random, and the
    grand product of the sorted columns is bit-exact against the oracle and returns to 1 on the last usable row"""
    import torch
    n = 1 << k
    usable = n - N_BLINDS - 1
    inp, tab, oi, ot = _check_permute(be, orc, *make_shape("spectre", usable, seed=k))
    tail = [orc.fr_random_chacha(n - usable, 920 + i) for i in range(4)]
    compressed = [np.concatenate([inp, tail[0]]), np.concatenate([tab, tail[1]])]
    permuted = [torch.cat([oi, _dev(torch, tail[2])]), torch.cat([ot, _dev(torch, tail[3])])]
    beta, gamma = orc.fr_random_chacha(2, 930)
    blinds = orc.fr_random_chacha(N_BLINDS, 931).reshape(-1, 4)
    z = _lookup_product(be, orc, compressed + permuted, beta, gamma, blinds)
    want = orc.lookup_product(*compressed, _host(permuted[0]), _host(permuted[1]), beta, gamma, blinds)
    assert np.array_equal(z, want)
    assert np.array_equal(z[usable], orc.fr([1])[0])
    assert np.array_equal(z[n - N_BLINDS:], blinds)
