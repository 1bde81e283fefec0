"""GPU: the three chunked scans of csrc/poly.cu (grand product, Kate division, batch inversion), spb_product_dev, the
Horner and weighted folds, and the argument provers of csrc/plonk.cu built on them (spb_permutation_product_dev, the
SHPLONK opener), at the row counts that reach each branch of their carry passes and at their documented limits; and the
lifecycle of the SHPLONK handle (slots or its own buffers, abort, finish on error, release_workspace). Every result is
bit-exact against the serial recurrence in Python integers up to PY_REFERENCE_MAX rows and against the C oracle beyond."""
import ctypes

import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be  # noqa: F401

pytestmark = pytest.mark.gpu

R = pyref.R_MOD
RINV = pow(1 << 256, -1, R)
PY_REFERENCE_MAX = 1 << 17

# Restated from spectre_b200/csrc/poly.cu: the scans walk 64-row chunks (kScanChunk, kChunk); the grand product's carry
# pass (carry_product_kernel) and spb_product_dev's fold (total_product_kernel) run one block of 1024 threads, the Kate
# division's (carry_kate_kernel) one block of 512. Thread t of a carry block owns the chunk partials [t * per, (t + 1) * per),
# per = ceil(m / threads) for m chunks. Every size below is derived from these, so a changed constant renames a shape.
CHUNK = 64
PRODUCT_THREADS = 1024
KATE_THREADS = 512


def rows(m, last=CHUNK):
    """row count of m chunks whose last chunk holds `last` rows"""
    return (m - 1) * CHUNK + last


def _dev(torch, arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _ints(arr):
    """(n, 4) Montgomery limbs -> canonical Python ints"""
    raw = np.ascontiguousarray(arr, dtype=np.uint64).tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") * RINV % R for i in range(0, len(raw), 32)]


def _random(be, orc, n, seed):
    """n ChaCha20 Fr draws; long columns are drawn on the device (spb_fr_random_chacha_dev, the same stream as the oracle's,
    tests/test_gpu_poly.py) because the CPU keystream would dominate the run time"""
    if n < 1 << 16:
        return orc.fr_random_chacha(n, 0x5ca40000 + seed)
    import torch
    out = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    be.fr_random_chacha_dev(0x5ca40000 + seed, 0, out.data_ptr(), n)
    return _host(out)


@pytest.fixture(scope="module", autouse=True)
def _free_module_buffers(be):
    """The 2^23- and 2^24-row scans grow the session context's workspaces and torch's cached blocks by several GiB; give
    them back so that later modules can prove at K = 24 on the same device."""
    yield
    import torch
    _PARAMS.clear()
    torch.cuda.synchronize()
    be.release_workspace()
    torch.cuda.empty_cache()


# ---- grand product ------------------------------------------------------------------------------------------------
def _grand_product_reference(orc, a, init):
    """z[0] = init, z[i + 1] = z[i] * a[i]: Python integers, or the oracle's lookup product with only the compressed input
    in the numerator (beta = gamma = 0, every other column 1) beyond PY_REFERENCE_MAX rows"""
    n = a.shape[0]
    if n <= PY_REFERENCE_MAX:
        z, acc = [], orc.fr_ints(init.reshape(1, 4))[0]
        for v in _ints(a):
            z.append(acc)
            acc = acc * v % R
        return orc.fr(z)
    ones = np.broadcast_to(orc.fr([1]), (n, 4)).copy()
    zero = np.zeros(4, np.uint64)
    z = orc.lookup_product(a, ones, ones, ones, zero, zero, np.zeros((0, 4), np.uint64))
    return orc.vec_scale(z, init)


def _product_shape(m, last=CHUNK):
    per = -(-m // PRODUCT_THREADS)
    return pytest.param(rows(m, last), id="m%d_per%d%s" % (m, per, "" if last == CHUNK else "_short_last_chunk"))


GRAND_PRODUCT_SHAPES = [
    pytest.param(1, id="one_row"),
    pytest.param(CHUNK, id="m1_one_chunk"),
    _product_shape(PRODUCT_THREADS - 1),
    _product_shape(PRODUCT_THREADS - 1, 1),
    pytest.param(rows(PRODUCT_THREADS), id="m_eq_blockDim"),
    _product_shape(PRODUCT_THREADS + 1, 1),                     # per 2: thread 512 holds one chunk of two
    _product_shape(2 * PRODUCT_THREADS),
    _product_shape(2 * PRODUCT_THREADS + 1, CHUNK - 5),         # per 3: threads 683.. start past m
    pytest.param(rows(3 * PRODUCT_THREADS - 1), id="per3_partial_last_thread"),
    _product_shape(3 * PRODUCT_THREADS + 1),
    pytest.param(1 << 22, id="m65536_per64"),
    pytest.param((1 << 22) + 1, id="m65537_per65_short_last_chunk"),
    pytest.param((1 << 23) - 1, id="m131072_per128_short_last_chunk"),
    pytest.param(1 << 23, id="m131072_per128"),
    pytest.param(1 << 24, id="m262144_per256", marks=pytest.mark.slow),
]


@pytest.mark.parametrize("n", GRAND_PRODUCT_SHAPES)
def test_grand_product(be, orc, n):
    """spb_grand_product_dev (init 1) and spb_grand_product_seeded_dev with a random and a zero seed"""
    import torch
    a = _random(be, orc, n, n % 1000003)
    da = _dev(torch, a)
    dz = torch.empty_like(da)
    be.grand_product_dev(da.data_ptr(), n, dz.data_ptr())
    one = orc.fr([1])[0]
    want = _grand_product_reference(orc, a, one)
    assert np.array_equal(_host(dz), want), "grand product"
    seed = _random(be, orc, 1, 7)[0]
    be.grand_product_seeded_dev(da.data_ptr(), n, seed, dz.data_ptr())
    assert np.array_equal(_host(dz), orc.vec_scale(want, seed)), "seeded grand product"
    be.grand_product_seeded_dev(da.data_ptr(), n, np.zeros(4, np.uint64), dz.data_ptr())
    assert not _host(dz).any(), "zero seed"


ZERO_ROWS = {"first_row": [0], "row63": [CHUNK - 1], "row64": [CHUNK], "last_row": [-1], "zero_chunk": list(range(5 * CHUNK, 6 * CHUNK))}


@pytest.mark.parametrize("where", sorted(ZERO_ROWS))
def test_grand_product_through_zeros(be, orc, where):
    """a zero factor zeroes every later row and no earlier one, across the chunk and carry-slice boundaries (m = 2049, per 3)"""
    import torch
    n = rows(2 * PRODUCT_THREADS + 1, CHUNK - 5)
    a = _random(be, orc, n, 11)
    a[ZERO_ROWS[where]] = 0
    seed = _random(be, orc, 1, 12)[0]
    da = _dev(torch, a)
    dz = torch.empty_like(da)
    be.grand_product_seeded_dev(da.data_ptr(), n, seed, dz.data_ptr())
    got = _host(dz)
    assert np.array_equal(got, _grand_product_reference(orc, a, seed))
    first = ZERO_ROWS[where][0] % n
    assert not got[first + 1:].any() and all(got[:first + 1].any(axis=1))


def _total_shape(m, last=CHUNK):
    return pytest.param(rows(m, last), id="m%d_stride_iters%d" % (m, -(-m // PRODUCT_THREADS)))


@pytest.mark.parametrize("n", [pytest.param(0, id="empty"), pytest.param(1, id="one_row"), _total_shape(1000, 17), _total_shape(PRODUCT_THREADS),
                               _total_shape(PRODUCT_THREADS + 1, 1), _total_shape(3 * PRODUCT_THREADS + 5), _total_shape(1 << 16)])
def test_product(be, orc, n):
    """spb_product_dev: the product of all rows, folded by total_product_kernel's stride loop (64 passes at 2^16 chunks);
    n = 0 gives 1"""
    import torch
    if n == 0:
        assert orc.fr_ints(be.product_dev(0, 0).reshape(1, 4)) == [1]
        return
    a = _random(be, orc, n, 20 + n % 1000)
    da = _dev(torch, a)
    got = orc.fr_ints(be.product_dev(da.data_ptr(), n).reshape(1, 4))[0]
    if n <= PY_REFERENCE_MAX:
        want = 1
        for v in _ints(a):
            want = want * v % R
    else:
        want = orc.fr_ints(_grand_product_reference(orc, np.concatenate([a, orc.fr([1])]), orc.fr([1])[0])[-1:])[0]
    assert got == want


# ---- Kate division ------------------------------------------------------------------------------------------------
def _kate_reference(orc, a, b):
    """q[i] = a[i + 1] + b q[i + 1], q[n - 2] = a[n - 1]"""
    n = a.shape[0]
    if n > PY_REFERENCE_MAX:
        return orc.kate_division(a, b)
    ai, bi = _ints(a), orc.fr_ints(np.asarray(b).reshape(1, 4))[0]
    q, t = [0] * (n - 1), 0
    for i in range(n - 2, -1, -1):
        t = (ai[i + 1] + bi * t) % R
        q[i] = t
    return orc.fr(q)


def _kate_shape(m, last=CHUNK, name=None):
    per = -(-m // KATE_THREADS)
    return pytest.param(rows(m, last) + 1, id=name or "m%d_per%d%s" % (m, per, "" if last == CHUNK else "_short_last_chunk"))


KATE_SHAPES = [
    pytest.param(2, id="one_quotient_row"),
    _kate_shape(KATE_THREADS - 1),
    _kate_shape(KATE_THREADS, name="m_eq_blockDim"),
    _kate_shape(KATE_THREADS + 1),
    _kate_shape(KATE_THREADS + 1, 1),
    _kate_shape(2 * KATE_THREADS),
    _kate_shape(2 * KATE_THREADS + 1, 2),
    _kate_shape(3 * KATE_THREADS),
    _kate_shape(3 * KATE_THREADS + 1, name="per4_partial_last_thread"),
    pytest.param((1 << 23) + 1, id="shplonk_k23"),
    pytest.param(1 << 24, id="shplonk_k24", marks=pytest.mark.slow),
]


@pytest.mark.parametrize("n", KATE_SHAPES)
def test_kate_division(be, orc, n):
    import torch
    a = _random(be, orc, n, 30 + n % 1000)
    b = _random(be, orc, 1, 31)[0]
    da = _dev(torch, a)
    dq = torch.empty((n - 1, 4), dtype=torch.int64, device="cuda")
    be.kate_division_dev(da.data_ptr(), n, b, dq.data_ptr())
    assert np.array_equal(_host(dq), _kate_reference(orc, a, b))


def _special_points():
    w64 = pyref.omega(6)                                        # b^64 = 1: the chunk multiplier b_chunk is one
    return {"zero": 0, "one": 1, "minus_one": R - 1, "root64": w64, "root64_inverse": pow(w64, -1, R), "omega16_pow5": pow(pyref.omega(16), 5, R),
            "omega20_pow77777": pow(pyref.omega(20), 77777, R)}


@pytest.mark.parametrize("point", sorted(_special_points()))
def test_kate_division_at_special_points(be, orc, point):
    """b = 0, 1, -1, a primitive 64th root of unity (b_chunk = 1) and roots of unity of the domains, at m = 1025 (per 3)"""
    import torch
    n = rows(2 * KATE_THREADS + 1, 2) + 1
    a = _random(be, orc, n, 40)
    b = orc.fr([_special_points()[point]])[0]
    da = _dev(torch, a)
    dq = torch.empty((n - 1, 4), dtype=torch.int64, device="cuda")
    be.kate_division_dev(da.data_ptr(), n, b, dq.data_ptr())
    assert np.array_equal(_host(dq), _kate_reference(orc, a, b))


@pytest.mark.parametrize("point", ["random", "root64", "omega16_pow5"])
def test_kate_division_of_an_exact_multiple(be, orc, point):
    """a = (X - b) r(X): the quotient is r, and q (X - b) = a in Python integers"""
    import torch
    n = rows(2 * KATE_THREADS + 1, 2) + 1
    ri = _ints(_random(be, orc, n - 1, 41))
    bi = orc.fr_ints(_random(be, orc, 1, 42))[0] if point == "random" else _special_points()[point]
    ai = [(-bi * ri[0]) % R] + [(ri[i - 1] - bi * ri[i]) % R for i in range(1, n - 1)] + [ri[n - 2]]
    a = orc.fr(ai)
    da = _dev(torch, a)
    dq = torch.empty((n - 1, 4), dtype=torch.int64, device="cuda")
    be.kate_division_dev(da.data_ptr(), n, orc.fr([bi])[0], dq.data_ptr())
    qi = _ints(_host(dq))
    assert qi == ri
    assert [(-bi * qi[0]) % R] + [(qi[i - 1] - bi * qi[i]) % R for i in range(1, n - 1)] + [qi[n - 2]] == ai


# ---- batch inversion ----------------------------------------------------------------------------------------------
def _batch_invert_check(orc, a, got):
    """zeros stay zero, every other element is its inverse (Python integers up to PY_REFERENCE_MAX rows), and the oracle agrees"""
    assert np.array_equal(got, orc.batch_invert(a))
    if a.shape[0] <= PY_REFERENCE_MAX:
        assert _ints(got) == [pow(v, -1, R) if v else 0 for v in _ints(a)]


def _zero_pattern(name, n):
    m = -(-n // CHUNK)
    return {"chunk_edges": [0, 2 * CHUNK - 1, 2 * CHUNK, 3 * CHUNK - 1, 4 * CHUNK, n - 1],
            "first_chunk": list(range(CHUNK)),
            "last_chunk": list(range((m - 1) * CHUNK, n)),
            "middle_chunks": list(range(7 * CHUNK, 9 * CHUNK)),
            "every_other_row": list(range(1, n, 2))}[name]


@pytest.mark.parametrize("pattern", ["chunk_edges", "first_chunk", "last_chunk", "middle_chunks", "every_other_row"])
def test_batch_invert_with_zeros(be, orc, pattern):
    """zeros on a chunk's first or last row and whole zero chunks, at m = 1025 chunks with a one-row last chunk"""
    import torch
    n = rows(PRODUCT_THREADS + 1, 1)
    a = _random(be, orc, n, 50)
    a[_zero_pattern(pattern, n)] = 0
    da = _dev(torch, a)
    be.batch_invert_dev(da.data_ptr(), n)
    _batch_invert_check(orc, a, _host(da))


@pytest.mark.parametrize("case", ["all_zero", "single_nonzero", "ones_and_minus_ones"])
def test_batch_invert_special_values(be, orc, case):
    import torch
    n = rows(37, 9)
    if case == "all_zero":
        a = np.zeros((n, 4), np.uint64)
    elif case == "single_nonzero":
        a = np.zeros((n, 4), np.uint64); a[5 * CHUNK + 17] = _random(be, orc, 1, 51)[0]
    else:
        a = orc.fr([1 if i % 3 else R - 1 for i in range(n)])
    da = _dev(torch, a)
    be.batch_invert_dev(da.data_ptr(), n)
    _batch_invert_check(orc, a, _host(da))


@pytest.mark.parametrize("n", [pytest.param((1 << 22) + 1, id="m65537_short_last_chunk"), pytest.param(1 << 24, id="m262144", marks=pytest.mark.slow)])
def test_batch_invert_large(be, orc, n):
    import torch
    a = _random(be, orc, n, 52)
    a[[0, CHUNK, n // 2, n - 1]] = 0
    a[(n // 3) & ~(CHUNK - 1):((n // 3) & ~(CHUNK - 1)) + CHUNK] = 0
    da = _dev(torch, a)
    be.batch_invert_dev(da.data_ptr(), n)
    _batch_invert_check(orc, a, _host(da))


# ---- Horner and weighted folds ------------------------------------------------------------------------------------
FOLD_ROWS = 4 * 256 - 23                                        # not a multiple of the 256-thread blocks


@pytest.fixture(scope="module")
def fold_polys(be, orc):
    polys = [_random(be, orc, FOLD_ROWS, 100 + p) for p in range(153)]  # 153: the opened-query count of the sync-step shape
    return polys, [_ints(p) for p in polys]


@pytest.mark.parametrize("count", [1, 2, 153])
@pytest.mark.parametrize("y", ["zero", "one", "random"])
def test_lincomb(be, orc, fold_polys, count, y):
    """out = sum_p y^p polys[p] (Horner from the last polynomial down)"""
    import torch
    polys, pi = fold_polys
    yi = {"zero": 0, "one": 1, "random": orc.fr_ints(_random(be, orc, 1, 60))[0]}[y]
    d = [_dev(torch, p) for p in polys[:count]]
    out = torch.empty((FOLD_ROWS, 4), dtype=torch.int64, device="cuda")
    be.lincomb_dev([t.data_ptr() for t in d], orc.fr([yi])[0], out.data_ptr(), FOLD_ROWS)
    yp = [pow(yi, p, R) for p in range(count)]
    assert _ints(_host(out)) == [sum(yp[p] * pi[p][i] for p in range(count)) % R for i in range(FOLD_ROWS)]


@pytest.mark.parametrize("count", [1, 153])
@pytest.mark.parametrize("weights", ["zero", "one", "random"])
def test_weighted_sum(be, orc, fold_polys, count, weights):
    import torch
    polys, pi = fold_polys
    wi = {"zero": [0] * count, "one": [1] * count, "random": _ints(_random(be, orc, count, 61))}[weights]
    d = [_dev(torch, p) for p in polys[:count]]
    out = torch.empty((FOLD_ROWS, 4), dtype=torch.int64, device="cuda")
    be.weighted_sum_dev([t.data_ptr() for t in d], orc.fr(wi), out.data_ptr(), FOLD_ROWS)
    assert _ints(_host(out)) == [sum(wi[p] * pi[p][i] for p in range(count)) % R for i in range(FOLD_ROWS)]


# ---- permutation product ------------------------------------------------------------------------------------------
MAX_SET_COLS = 16                                               # kMaxSetCols in csrc/quotient.cuh


@pytest.mark.parametrize("k,sets,n_blinds", [
    pytest.param(16, [(144, MAX_SET_COLS), (160, MAX_SET_COLS)], 6, id="k16_two_full_sets_first_col160"),
    pytest.param(17, [(0, MAX_SET_COLS), (16, 5)], 0, id="k17_block_row_past_2^16"),
    pytest.param(17, [(3, 2)], "n-1", id="k17_all_rows_blinded"),
    pytest.param(20, [(100, 4), (104, 1)], 6, id="k20"),
    pytest.param(23, [(0, 2)], 6, id="k23", marks=pytest.mark.slow),
])
def test_permutation_product(be, orc, k, sets, n_blinds):
    """chained sets carrying last_z, up to 16 columns per set and first_col 160, against the oracle's permutation::commit"""
    import torch
    n = 1 << k
    n_blinds = n - 1 if n_blinds == "n-1" else n_blinds
    beta, gamma = _random(be, orc, 2, 70 + k)
    dz = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    last_o = last_g = orc.fr([1])[0]
    for s, (first_col, n_cols) in enumerate(sets):
        values = [_random(be, orc, n, 1000 * s + 2 * c) for c in range(n_cols)]
        sigma = [_random(be, orc, n, 1000 * s + 2 * c + 1) for c in range(n_cols)]
        values[0][3] = 0; sigma[-1][n - 5] = 0
        blinds = _random(be, orc, n_blinds, 80 + s).reshape(-1, 4)
        z_want, last_o = orc.permutation_product(k, values, sigma, first_col, beta, gamma, blinds, last_o)
        dv, ds = [_dev(torch, a) for a in values], [_dev(torch, a) for a in sigma]
        last_g = be.permutation_product_dev(k, [t.data_ptr() for t in dv], [t.data_ptr() for t in ds], first_col, beta, gamma, blinds, last_g, dz.data_ptr())
        assert np.array_equal(_host(dz), z_want), "set %d" % s
        assert np.array_equal(last_g, last_o.reshape(4)), "set %d" % s
        del dv, ds


def test_permutation_product_of_a_real_permutation_closes_at_k17(be, orc):
    """sigma encoding a permutation of equal cells over all 2^17 rows of three columns: the product returns to 1"""
    import torch
    k, n_cols = 17, 3
    n = 1 << k
    delta = orc.fr_ints(orc.fr_delta().reshape(1, 4))[0]
    omega = pyref.omega(k)
    opow = [1] * n
    for i in range(1, n):
        opow[i] = opow[i - 1] * omega % R
    ident = [[pow(delta, c, R) * w % R for w in opow] for c in range(n_cols)]
    vals = [[(7 * i + c) % 50 for i in range(n)] for c in range(n_cols)]
    cells = {}
    for c in range(n_cols):
        for i in range(n):
            cells.setdefault(vals[c][i], []).append((c, i))
    sig = [[0] * n for _ in range(n_cols)]
    for group in cells.values():                                # one cycle per value class
        for a, b in zip(group, group[1:] + group[:1]):
            sig[a[0]][a[1]] = ident[b[0]][b[1]]
    values = [orc.fr(v) for v in vals]; sigma = [orc.fr(s) for s in sig]
    beta, gamma = _random(be, orc, 2, 90)
    dv, ds = [_dev(torch, a) for a in values], [_dev(torch, a) for a in sigma]
    dz = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    last = be.permutation_product_dev(k, [t.data_ptr() for t in dv], [t.data_ptr() for t in ds], 0, beta, gamma, np.zeros((0, 4), np.uint64), orc.fr([1])[0],
                                      dz.data_ptr())
    z = _host(dz)
    z_want, _ = orc.permutation_product(k, values, sigma, 0, beta, gamma, np.zeros((0, 4), np.uint64), orc.fr([1])[0])
    assert np.array_equal(z, z_want)
    b, g = orc.fr_ints(np.stack([beta, gamma]))
    num = den = 1
    for c in range(n_cols):                                     # z[n-1] times the last row's factor is 1
        num = num * (vals[c][n - 1] + b * ident[c][n - 1] + g) % R
        den = den * (vals[c][n - 1] + b * sig[c][n - 1] + g) % R
    assert _ints(z[n - 1:n])[0] * num % R == den
    assert np.array_equal(last, z[n - 1])


def test_permutation_product_rejects_seventeen_columns(be, orc):
    import torch
    from spectre_b200.halo2 import BackendError
    k = 6
    col = _dev(torch, _random(be, orc, 1 << k, 91))
    dz = torch.empty_like(col)
    beta, gamma = _random(be, orc, 2, 92)
    with pytest.raises(BackendError, match="columns per set"):
        be.permutation_product_dev(k, [col.data_ptr()] * (MAX_SET_COLS + 1), [col.data_ptr()] * (MAX_SET_COLS + 1), 0, beta, gamma, np.zeros((0, 4), np.uint64),
                                   orc.fr([1])[0], dz.data_ptr())
    be.permutation_product_dev(k, [col.data_ptr()] * MAX_SET_COLS, [col.data_ptr()] * MAX_SET_COLS, 0, beta, gamma, np.zeros((0, 4), np.uint64), orc.fr([1])[0],
                               dz.data_ptr())


# ---- SHPLONK ------------------------------------------------------------------------------------------------------
MAX_POINTS = 8                                                  # points per rotation set (spb_rotation_set, SmallPoly in csrc/plonk.cu)


class _Opening:
    """rotation sets over random polynomials kept on the device: layout = [(points as ints, poly ids)], one polynomial per id"""

    def __init__(self, be, orc, k, layout, seed):
        import torch
        self.n = 1 << k
        ids = sorted({p for _, pids in layout for p in pids}, key=str)
        self.host = {p: _random(be, orc, self.n, seed * 1000 + i) for i, p in enumerate(ids)}
        self.dev = {p: _dev(torch, a) for p, a in self.host.items()}
        self.sets = []
        for pts, pids in layout:
            P = orc.fr(pts)
            ev = np.stack([np.stack([orc.eval_polynomial(self.host[p], x) for x in P]) for p in pids])
            self.sets.append((P, pids, ev))

    def host_sets(self):
        return [(P, [self.host[p] for p in pids], ev) for P, pids, ev in self.sets]

    def dev_sets(self):
        return [(P, [self.dev[p].data_ptr() for p in pids], ev) for P, pids, ev in self.sets]

    def expected(self, orc, y, v, u):
        h_x = orc.shplonk_quotient(self.n, self.host_sets(), y, v)
        return orc.commit_known_tau(h_x), orc.commit_known_tau(orc.shplonk_linearisation(self.n, self.host_sets(), y, v, u, h_x))


_PARAMS = {}


def _params(be, orc, k):
    """the seed-0 SRS of 2^k points, set up once per module (dropped at its teardown)"""
    from spectre_b200.halo2 import ParamsKZG
    if k not in _PARAMS:
        _PARAMS[k] = ParamsKZG.setup(be, k, orc.srs_tau())
    return _PARAMS[k]


def _open_and_check(be, orc, k, op, seed):
    y, v, u = _random(be, orc, 3, seed)
    want_h, want_final = op.expected(orc, y, v, u)
    h, handle = be.shplonk_begin_dev(_params(be, orc, k), op.n, op.dev_sets(), y, v)
    got = be.shplonk_finish_dev(handle, u)
    assert np.array_equal(orc.g1_to_affine(h), want_h)
    assert np.array_equal(orc.g1_to_affine(got), want_final)


@pytest.mark.parametrize("k", [7, 12])
def test_shplonk_eight_point_set(be, orc, k):
    """one set of 8 points: eight chained Kate divisions of lengths n .. n - 7 (the last chunk shrinks from 63 quotient rows to
    56); beside it a one-point set. The subtracted R(X) has 8 coefficients here, but no output depends on them: R has degree
    < 8 and each of the eight divisions drops the constant coefficient of its dividend."""
    pts = _ints(_random(be, orc, MAX_POINTS + 1, 200 + k))
    op = _Opening(be, orc, k, [(pts[:MAX_POINTS], ["a", "b", "c"]), (pts[MAX_POINTS:], ["d"])], 201 + k)
    _open_and_check(be, orc, k, op, 202 + k)


def test_shplonk_point_limits(be, orc):
    """9 points in a set are refused; at n = 8, 7 points are accepted and 8 refused (n_points < n)"""
    from spectre_b200.halo2 import BackendError
    pts = _ints(_random(be, orc, MAX_POINTS + 1, 210))
    big = _Opening(be, orc, 6, [(pts, ["a"])], 211)
    y, v = _random(be, orc, 2, 212)
    with pytest.raises(BackendError, match="malformed"):
        be.shplonk_begin_dev(_params(be, orc, 6), big.n, big.dev_sets(), y, v)
    small = _Opening(be, orc, 3, [(pts[:7], ["a", "b"])], 213)
    _open_and_check(be, orc, 3, small, 214)
    eight = _Opening(be, orc, 3, [(pts[:8], ["a"])], 215)
    with pytest.raises(BackendError, match="malformed"):
        be.shplonk_begin_dev(_params(be, orc, 3), eight.n, eight.dev_sets(), y, v)
    be.release_workspace()                                      # no handle was left open by the refusals


def _halo2lib_layout(k, x):
    """the rotation sets of the halo2lib sync-step shape: create_proof's multi-open query list (advice, permutation z,
    lookups, fixed, sigma, vanishing) through plonk.rotation_sets"""
    from spectre_b200 import circuits, plonk
    cs = circuits.halo2lib_shape()
    w, bf = pyref.omega(k), cs.blinding_factors()
    n_sets = -(-len(cs.permutation) // cs.chunk_len())
    q = [(("advice", c), r) for c, r in cs.advice_queries]
    for s in range(n_sets):
        q += [(("perm", s), 0), (("perm", s), 1)]
    q += [(("perm", s), -(bf + 1)) for s in reversed(range(n_sets - 1))]
    for li in range(len(cs.lookups)):
        q += [(("lk_z", li), 0), (("lk_a", li), 0), (("lk_s", li), 0), (("lk_a", li), -1), (("lk_z", li), 1)]
    q += [(("fixed", c), r) for c, r in cs.fixed_queries]
    q += [(("sigma", c), 0) for c in range(len(cs.permutation))]
    q += [(("h",), 0), (("random",), 0)]
    sets = plonk.rotation_sets([(pid, x * pow(w, r, R) % R, 0) for pid, r in q])
    return [(list(pts), list(pids)) for pts, pids, _ in sets]


def test_shplonk_halo2lib_rotation_sets_at_k16(be, orc):
    k = 16
    x = orc.fr_ints(_random(be, orc, 1, 220))[0]
    layout = _halo2lib_layout(k, x)
    assert len(layout) >= 4 and max(len(p) for p, _ in layout) >= 4
    _open_and_check(be, orc, k, _Opening(be, orc, k, layout, 221), 222)


def test_shplonk_polynomial_in_several_sets_with_reordered_points(be, orc):
    p = _ints(_random(be, orc, 5, 230))
    layout = [([p[0], p[1], p[2]], ["a", "b"]), ([p[2], p[0]], ["a", "c"]), ([p[3], p[1], p[4], p[0]], ["b", "a"]), ([p[4]], ["c"])]
    _open_and_check(be, orc, 10, _Opening(be, orc, 10, layout, 231), 232)


# ---- the SHPLONK handle: slots, own buffers, abort, finish on error ------------------------------------------------
class _Handles:
    """opened handles of one test; those still open at its end are aborted so that a failure does not hold the slots"""

    def __init__(self, be):
        self.be, self.open = be, []

    def begin(self, orc, k, op, seed):
        y, v, u = _random(self.be, orc, 3, seed)
        want_h, want_final = op.expected(orc, y, v, u)
        h, handle = self.be.shplonk_begin_dev(_params(self.be, orc, k), op.n, op.dev_sets(), y, v)
        self.open.append(handle)
        assert np.array_equal(orc.g1_to_affine(h), want_h)
        return handle, u, want_final

    def finish(self, orc, opened):
        handle, u, want_final = opened
        self.open.remove(handle)
        assert np.array_equal(orc.g1_to_affine(self.be.shplonk_finish_dev(handle, u)), want_final)

    def abort(self, opened):
        self.open.remove(opened[0])
        self.be.shplonk_abort_dev(opened[0])

    def close(self):
        for handle in self.open:
            self.be.shplonk_abort_dev(handle)


@pytest.fixture
def handles(be):
    h = _Handles(be)
    yield h
    h.close()


def _ops(be, orc, k, count, seed):
    pts = _ints(_random(be, orc, 3, seed))
    return [_Opening(be, orc, k, [(pts[:2], ["a"]), (pts[1:], ["b", "c"])], seed + 1 + i) for i in range(count)]


def _workspace_free(be):
    from spectre_b200.halo2 import BackendError
    try:
        be.release_workspace()
        return True
    except BackendError as e:
        assert "handle is open" in str(e)
        return False


@pytest.mark.parametrize("order", ["first_opened_first", "second_opened_first"])
def test_shplonk_two_open_handles(be, orc, handles, order):
    """a second handle while the first holds the context's slots runs in its own cudaMalloc'd buffers"""
    k = 9
    a, b = _ops(be, orc, k, 2, 240)
    A = handles.begin(orc, k, a, 243)
    B = handles.begin(orc, k, b, 244)
    for h in ((A, B) if order == "first_opened_first" else (B, A)):
        handles.finish(orc, h)
    assert _workspace_free(be)


def test_shplonk_handle_sequence_keeps_the_slots_with_their_owner(be, orc, handles):
    """open A (slots), open B (own buffers), finish B, open C, finish A, finish C: finishing B must not hand A's slots to C"""
    k = 9
    a, b, c = _ops(be, orc, k, 3, 250)
    A = handles.begin(orc, k, a, 254)
    B = handles.begin(orc, k, b, 255)
    handles.finish(orc, B)
    C = handles.begin(orc, k, c, 256)
    handles.finish(orc, A)
    handles.finish(orc, C)
    assert _workspace_free(be)


def test_shplonk_abort_gives_the_slots_back(be, orc, handles):
    k = 8
    a, b = _ops(be, orc, k, 2, 260)
    A = handles.begin(orc, k, a, 263)
    assert not _workspace_free(be)
    handles.abort(A)
    assert _workspace_free(be)
    B = handles.begin(orc, k, b, 264)                           # the next handle takes the slots again
    C = handles.begin(orc, k, a, 265)                           # its own buffers
    assert not _workspace_free(be)
    handles.abort(C)
    handles.finish(orc, B)                                      # B's slots were left alone

    assert _workspace_free(be)


def test_shplonk_finish_with_a_bad_argument_consumes_the_handle(be, orc, handles):
    """include/spectre_b200.h: finish "consumes the handle (also on error)": a null u or commitment, and u on an opening point"""
    from spectre_b200.halo2 import BackendError
    k = 8
    (a,) = _ops(be, orc, k, 1, 270)
    out = np.empty(12, dtype=np.uint64)
    for bad in ("u", "commitment"):
        handle, u, _ = handles.begin(orc, k, a, 272)
        handles.open.remove(handle)                             # finish owns it from here on
        args = (None, out.ctypes.data_as(ctypes.c_void_p)) if bad == "u" else (u.ctypes.data_as(ctypes.c_void_p), None)
        assert be.lib.spb_shplonk_finish_dev(be.ctx, handle, *args) != 0
        assert b"null argument" in be.lib.spb_last_error(be.ctx)
        assert _workspace_free(be)
    handle, _, _ = handles.begin(orc, k, a, 273)
    handles.open.remove(handle)
    with pytest.raises(BackendError, match="opening points"):   # a point of set 1 that set 0 lacks: Z_{T \ S_0}(u) = 0
        be.shplonk_finish_dev(handle, a.sets[1][0][1])
    assert _workspace_free(be)
    handles.finish(orc, handles.begin(orc, k, a, 274))          # the context still opens normally


@pytest.mark.parametrize("exc", [RuntimeError, KeyboardInterrupt])
def test_create_proof_aborts_the_handle_when_the_transcript_raises(be, orc, exc):
    """an exception between shplonk_begin and shplonk_finish (the h commitment's transcript write) releases the handle: the
    workspace can be released, and the next proof is byte-identical to one made before"""
    from spectre_b200 import circuits, plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import FailingTranscript, SeededRng
    k, instances = 7, [3, 1, 4]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, lookup_bits=3, groups=20)
    E = plonk.DeviceEngine(be, _params(be, orc, k), k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    count = FailingTranscript(pk.vk_digest)
    before = plonk.create_proof(E, pk, [instances], [adv], SeededRng(9), count)
    with pytest.raises(exc, match="injected"):
        plonk.create_proof(E, pk, [instances], [adv], SeededRng(9), FailingTranscript(pk.vk_digest, count.points - 2, exc))
    be.release_workspace()
    assert plonk.create_proof(E, pk, [instances], [adv], SeededRng(9), EvmTranscriptWrite(pk.vk_digest)) == before
