"""Every field and G1 primitive of spectre_b200/csrc/{ptx,field,curve}.cuh on the device, through the spb_test_* hooks and
two production kernels.

  * the carry-covering corpus of tests/arith_corpus.py, per primitive and field: equal to Python integers and, limb for
    limb, to the emulated build of the same algorithm (libhostemu_ptx.so) -- the device runs the inline asm of ptx.cuh,
    which no CPU build compiles;
  * raw (non-Montgomery) limb patterns for mul, sqr and a*b - c*d;
  * 2^22 random operands per primitive against the independent 64-bit host algorithm (libhostemu_native.so);
  * the Fr corpus through spb_graph_evaluate_dev (one-calculation programs for add, sub, mul, sqr, dbl, neg) and
    spb_vec_mul_dev, whose kernels inline the same primitives under their own register allocation;
  * the exceptional cases of the XYZZ formulas with zz != 1, so equal points arrive in different representations.
"""
import random

import numpy as np
import pytest

from tests import arith_corpus as ac
from tests import pyref
from tests.gpu_common import be  # noqa: F401

pytestmark = pytest.mark.gpu
FIELDS = ("fr", "fq")
P = pyref.P_MOD


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """(directory of the corpus' trace build, emulated PTX build, 64-bit host build)"""
    d = tmp_path_factory.mktemp("hostemu_arith")
    return d, ac.build_hostemu(d, "ptx"), ac.build_hostemu(d, "native")


def _u64(limbs32):
    return np.ascontiguousarray(limbs32, dtype=np.uint32).view(np.uint64).reshape(-1, 4)


def _device(be, field, prim, tuples):
    """-> (n, 8) uint32 result limbs of the primitive on the device"""
    cols = [_u64(ac.limbs([t[i] for t in tuples])) for i in range(len(tuples[0]))]
    if prim == "mul_sub_mul":
        out = be.test_field_mul_sub_mul(field, *cols)
    else:
        out = be.test_field_op(field, prim, cols[0], cols[1] if len(cols) > 1 else None)
    return out.view(np.uint32).reshape(-1, 8)


def _host(lib, field, prim, tuples):
    return ac.run_host(lib, field, prim, tuples)


@pytest.mark.parametrize("field", FIELDS)
def test_corpus_on_the_device(be, emu, field):
    d, ptx, _ = emu
    for prim in ac.PRIMITIVES:
        tuples = ac.corpus(d, field, prim)
        got = _device(be, field, prim, tuples)
        assert ac.ints(got) == [ac.expected(field, prim, t) for t in tuples], (field, prim)
        assert np.array_equal(got, _host(ptx, field, prim, tuples)), (field, prim)


@pytest.mark.parametrize("field", FIELDS)
def test_unary_and_power_primitives(be, emu, field):
    """dbl, to_mont, inv, is_canonical, pow and pow_u64 on the special values and the unary corpora"""
    d, ptx, _ = emu
    m = ac.MODULI[field]
    vals = sorted(set(ac.special_values(m)) | {t[0] for prim in ("sqr", "neg", "from_mont") for t in ac.corpus(d, field, prim)})
    for prim in ("dbl", "to_mont", "inv"):
        tuples = [(v,) for v in vals]
        got = _device(be, field, prim, tuples)
        assert ac.ints(got) == [ac.expected(field, prim, t) for t in tuples], prim
        cols = [ac.limbs(vals), np.zeros((len(vals), 8), np.uint32)]
        host = np.empty_like(cols[0])
        ptx.he_field_op(ac.FIELD_CODE[field], ac.OPS[prim], ac._p(cols[0]), ac._p(cols[1]), ac._p(host), ac.ctypes.c_size_t(len(vals)))
        assert np.array_equal(got, host), prim
    # canonicity: every value of the corpus, and raw limbs at and above the modulus (limb by limb)
    ml = ac._limbs32(m)
    near = [m, m + 1, (1 << 256) - 1, m + (1 << 224)] + [m + (1 << (32 * j)) for j in range(8)]
    # m with limb i raised by one (above m), and m with limb i lowered by one and every limb below it all-ones (below m)
    near += [m - (ml[i] << (32 * i)) + (((ml[i] + 1) & 0xFFFFFFFF) << (32 * i)) for i in range(8)]
    near += [(m >> (32 * i) << (32 * i)) - (1 << (32 * i)) + ((1 << (32 * i)) - 1) for i in range(8) if ml[i]]
    cand = vals + [v for v in near if v < (1 << 256)]
    got = ac.ints(_device(be, field, "is_canonical", [(v,) for v in cand]))
    assert got == [1 if v < m else 0 for v in cand]
    # powers: a^e in Montgomery form is a^e R^(1-e) on raw limbs
    rng = random.Random(5)
    bases = [vals[i] for i in range(0, len(vals), max(1, len(vals) // 24))]
    rinv = ac.RINV[field]
    for prim, exps in (("pow", [0, 1, 2, 3, m - 2, m - 1, (1 << 256) - 1, rng.randrange(1 << 256)]),
                       ("pow_u64", [0, 1, 2, 3, 1 << 32, (1 << 63) | 1, (1 << 64) - 1, rng.randrange(1 << 64)])):
        tuples = [(b, e) for b in bases for e in exps]
        got = ac.ints(_device(be, field, prim, tuples))
        R = (1 << 256) % m
        assert got == [pow(b * rinv, e, m) * R % m for b, e in tuples], prim


@pytest.mark.parametrize("field", FIELDS)
def test_raw_limb_patterns(be, emu, field):
    """worst-case limb patterns handed over without Montgomery conversion: the result is a*b*2^-256 (sqr: a*a*2^-256)"""
    _, ptx, _ = emu
    m = ac.MODULI[field]
    vals = [m - 1 - i for i in range(16)] + [((1 << 254) - 1) % m, (1 << 224) - 1, m >> 1, (m >> 1) + 1]
    vals += [(0xFFFFFFFF << (32 * i)) % m for i in range(8)] + [((1 << (32 * i)) - 1) % m for i in range(1, 9)]
    pairs = [(a, b) for a in vals for b in vals]
    quads = [(a, b, c, e) for (a, b) in pairs[::7] for (c, e) in pairs[::31]]
    for prim, tuples in (("mul", pairs), ("sqr", [(v,) for v in vals]), ("mul_sub_mul", quads)):
        got = _device(be, field, prim, tuples)
        assert ac.ints(got) == [ac.expected(field, prim, t) for t in tuples], prim
        assert np.array_equal(got, _host(ptx, field, prim, tuples)), prim


def _random_limbs(m, n, seed):
    """n uniform-ish values below m as (n, 8) uint32 limbs: the top limb is drawn below the modulus' top limb"""
    g = np.random.default_rng(seed)
    x = g.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
    x[:, 7] = g.integers(0, m >> 224, size=n, dtype=np.uint64).astype(np.uint32)
    return x


@pytest.mark.parametrize("field", FIELDS)
def test_bulk_random_against_the_64bit_host_path(be, emu, field):
    _, _, native = emu
    n = 1 << 22
    m = ac.MODULI[field]
    cols = [_random_limbs(m, n, 100 * i + ac.FIELD_CODE[field]) for i in range(4)]
    c = ac.ctypes.c_size_t(n)
    for prim in ac.PRIMITIVES + ("dbl", "to_mont"):
        host = np.empty_like(cols[0])
        if prim == "mul_sub_mul":
            native.he_field_mul_sub_mul(ac.FIELD_CODE[field], *[ac._p(x) for x in cols], ac._p(host), c)
            got = be.test_field_mul_sub_mul(field, *[_u64(x) for x in cols])
        else:
            native.he_field_op(ac.FIELD_CODE[field], ac.OPS[prim], ac._p(cols[0]), ac._p(cols[1]), ac._p(host), c)
            got = be.test_field_op(field, prim, _u64(cols[0]), _u64(cols[1]))
        got = got.view(np.uint32).reshape(-1, 8)
        bad = np.nonzero((got != host).any(axis=1))[0]
        assert bad.size == 0, "%s %s: %d of %d differ, first at %d" % (field, prim, bad.size, n, bad[0])
    # spot-check the host path itself against Python integers
    idx = list(range(0, n, n // 64))
    a, b = ac.ints(cols[0][idx]), ac.ints(cols[1][idx])
    host = np.empty_like(cols[0])
    native.he_field_op(ac.FIELD_CODE[field], ac.OPS["mul"], ac._p(cols[0]), ac._p(cols[1]), ac._p(host), c)
    assert ac.ints(host[idx]) == [ac.expected(field, "mul", (x, y)) for x, y in zip(a, b)]


# ---- production kernels -------------------------------------------------------------------------------------------------
def _dev(torch, limbs32):
    return torch.from_numpy(_u64(limbs32).view(np.int64).copy()).cuda()


def test_fr_corpus_through_the_production_kernels(be, emu):
    """spb_graph_evaluate_dev with one-calculation programs (op 0..5: add, sub, mul, sqr, dbl, neg) and spb_vec_mul_dev"""
    import torch
    from tests.quotient_common import K_ADVICE
    d, _, _ = emu
    f = "fr"
    zero = np.zeros((1, 4), dtype=np.uint64)
    unary = sorted({t[0] for prim in ac.PRIMITIVES for t in ac.corpus(d, f, prim)})
    for op, prim in enumerate(("add", "sub", "mul", "sqr", "dbl", "neg")):
        tuples = ac.corpus(d, f, prim) if prim in ("add", "sub", "mul") else [(v,) for v in unary]
        if prim == "mul":
            tuples = tuples + [(t[0], 1) for t in ac.corpus(d, f, "from_mont")]
        size = 1 << max(1, (len(tuples) - 1).bit_length())
        a = np.zeros((size, 8), np.uint32); b = np.zeros((size, 8), np.uint32)
        a[:len(tuples)] = ac.limbs([t[0] for t in tuples])
        if op <= 2:
            b[:len(tuples)] = ac.limbs([t[1] for t in tuples])
        prog = np.array([op, 0, K_ADVICE, 0, K_ADVICE, 1] if op <= 2 else [op, 0, K_ADVICE, 0], dtype=np.uint32)
        da, db, dv = _dev(torch, a), _dev(torch, b), _dev(torch, np.zeros((size, 8), np.uint32))
        torch.cuda.synchronize()
        be.graph_evaluate_dev(prog, 1, 1, zero, np.array([0], np.int32), [], [da.data_ptr(), db.data_ptr()], [], zero, zero[0], zero[0], zero[0], zero[0],
                              dv.data_ptr(), size, 1)
        got = ac.ints(dv.cpu().numpy().view(np.uint64))[:len(tuples)]
        want = [ac.expected(f, prim, t) for t in tuples]
        assert got == want, prim
    tuples = ac.corpus(d, f, "mul") + [(t[0], 1) for t in ac.corpus(d, f, "from_mont")]
    da, db = _dev(torch, ac.limbs([t[0] for t in tuples])), _dev(torch, ac.limbs([t[1] for t in tuples]))
    torch.cuda.synchronize()
    be.vec_mul_dev(da.data_ptr(), db.data_ptr(), len(tuples))
    assert ac.ints(da.cpu().numpy().view(np.uint64)) == [ac.expected(f, "mul", t) for t in tuples]


# ---- G1 ---------------------------------------------------------------------------------------------------------------
R_Q = (1 << 256) % P
RINV_Q = pow(1 << 256, -1, P)


def _m(x):
    return x * R_Q % P


def _xyzz(pt, lam):
    """a point as XYZZ integers (x lam^2, y lam^3, lam^2, lam^3); None = the identity (zz = 0)"""
    if pt is None:
        return (0, 1, 0, 0)
    x, y = pt
    l2 = lam * lam % P
    l3 = l2 * lam % P
    return (x * l2 % P, y * l3 % P, l2, l3)


def _pack(rows):
    """rows of four integers (x, y, zz, zzz) -> (n, 16) uint64 of Montgomery limbs"""
    return _u64(ac.limbs([_m(v) for r in rows for v in r])).reshape(-1, 16)


def _raw_pack(rows):
    """rows of four raw limb integers (no Montgomery conversion)"""
    return _u64(ac.limbs([v for r in rows for v in r])).reshape(-1, 16)


def _unpack(arr):
    v = ac.ints(np.ascontiguousarray(arr).view(np.uint32).reshape(-1, 8))
    return [tuple(x * RINV_Q % P for x in v[4 * i:4 * i + 4]) for i in range(len(v) // 4)]


def _affine(row):
    x, y, zz, zzz = row
    if zz == 0:
        return None
    return (x * pow(zz, -1, P) % P, y * pow(zzz, -1, P) % P)


def _neg(pt):
    return None if pt is None else (pt[0], -pt[1] % P)


def _curve(be, ptx, op, p, q=None, k=None, raw=False):
    """the device result and the emulated build's, which must be the same limbs"""
    pk = (_raw_pack if raw else _pack)(p)
    qk = np.zeros_like(pk) if q is None else _pack(q)
    got = be.test_curve_op(op, pk, qk, k)
    host = np.empty_like(got)
    kk = None if k is None else np.ascontiguousarray(k, dtype=np.uint32)
    ptx.he_curve_op(be.TEST_CURVE_OPS[op], ac._p(pk), ac._p(qk), None if kk is None else ac._p(kk), ac._p(host), ac.ctypes.c_size_t(len(p)))
    assert np.array_equal(got, host), op
    return _unpack(got), got


def test_curve_exceptional_cases(be, emu):
    _, ptx, _ = emu
    rng = random.Random(17)
    G = (1, 2)
    pts = [G] + [pyref.ec_mul(G, rng.randrange(1, pyref.R_MOD)) for _ in range(6)]
    lam = lambda: rng.randrange(2, P)
    ident = (0, 1, 0, 0)
    # acc (XYZZ, zz != 1) + q (affine): P + P (doubling branch), P + (-P), identity on either side, affine (0, 0), generic sums
    p_rows, q_rows, want = [], [], []
    for i, pt in enumerate(pts):
        other = pts[(i + 1) % len(pts)]
        for acc, q, w in ((pt, pt, pyref.ec_add(pt, pt)), (pt, _neg(pt), None), (None, pt, pt), (pt, None, pt), (pt, other, pyref.ec_add(pt, other))):
            p_rows.append(_xyzz(acc, lam())); want.append(w)
            q_rows.append((0, 0, 0, 0) if q is None else (q[0], q[1], 0, 0))
    got, _ = _curve(be, ptx, "add_mixed", p_rows, q_rows)
    assert [_affine(r) for r in got] == want
    # XYZZ + XYZZ, both in their own representation
    p_rows, q_rows, want = [], [], []
    for i, pt in enumerate(pts):
        other = pts[(i + 2) % len(pts)]
        for acc, q, w in ((pt, pt, pyref.ec_add(pt, pt)), (pt, _neg(pt), None), (None, pt, pt), (pt, None, pt), (None, None, None),
                          (pt, other, pyref.ec_add(pt, other))):
            p_rows.append(_xyzz(acc, lam())); q_rows.append(_xyzz(q, lam())); want.append(w)
    got, _ = _curve(be, ptx, "add", p_rows, q_rows)
    assert [_affine(r) for r in got] == want
    # doublings, to_affine, identity
    rows = [_xyzz(pt, lam()) for pt in pts] + [ident]
    got, _ = _curve(be, ptx, "dbl", rows)
    assert [_affine(r) for r in got] == [pyref.ec_add(pt, pt) for pt in pts] + [None]
    got, _ = _curve(be, ptx, "dbl_affine", [(pt[0], pt[1], 0, 0) for pt in pts])
    assert [_affine(r) for r in got] == [pyref.ec_add(pt, pt) for pt in pts]
    got, _ = _curve(be, ptx, "to_affine", rows)
    assert [r[:2] for r in got] == [pt for pt in pts] + [(0, 0)]
    assert all(r[2:] == (0, 0) for r in got)
    # k * P for the small scalars the MSM's window code uses
    ks = [0, 1, 2, 3, 1 << 16, (1 << 32) - 1, rng.randrange(1 << 32)]
    rows = [_xyzz(pt, lam()) for pt in pts[:3] for _ in ks] + [ident] * 2
    kk = ks * 3 + [0, 5]
    got, _ = _curve(be, ptx, "mul_u32", rows, k=kk)
    assert [_affine(r) for r in got] == [pyref.ec_mul(pt, k) for pt in pts[:3] for k in ks] + [None, None]


def test_affine_check_verdicts(be, emu):
    """valid points and the identity pass; non-canonical x, non-canonical y, both (x is reported first), off the curve"""
    _, ptx, _ = emu
    G = (1, 2)
    Q = pyref.ec_mul(G, 12345)
    mx = lambda v: _m(v)
    cases = [((mx(G[0]), mx(G[1])), 0), ((mx(Q[0]), mx(Q[1])), 0), ((0, 0), 0),
             ((mx(G[0]) + P, mx(G[1])), 1), ((P, mx(G[1])), 1), (((1 << 256) - 1, mx(G[1])), 1),
             ((mx(G[0]), mx(G[1]) + P), 2), ((mx(G[0]), P), 2), ((0, P), 2),
             ((P, P), 1), ((mx(G[0]) + P, (1 << 256) - 1), 1),
             ((mx(G[0]), mx(G[1] + 1)), 3), ((mx(Q[0]), mx(-Q[1] % P + 1)), 3), ((0, mx(1)), 3), ((mx(1), 0), 3)]
    _, got = _curve(be, ptx, "affine_check", [(x, y, 0, 0) for (x, y), _ in cases], raw=True)
    verdicts = [int(v) for v in got.view(np.uint32).reshape(-1, 32)[:, 0]]
    assert verdicts == [w for _, w in cases]
