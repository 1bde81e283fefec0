"""CPU: a Python restatement of lookup::prover::permute_expression_pair, the properties the lookup argument needs of its
permuted columns, and the column shapes that drive the device sort (tests/test_gpu_lookup_shapes.py) through each branch of
its radix sort and of its leftover hand-out.

The restatement is checked here against the oracle on every shape at sizes up to 2^14, error cases included, so the GPU
tests can compare the device with the oracle at sizes where Python is too slow.

A shape is (pool, input_idx, table_idx): a list of distinct canonical integers and two index arrays into it. Only the pool
is converted to Montgomery form, so a 2^24-row column costs a numpy gather."""
import random
from collections import Counter

import numpy as np
import pytest

from tests import pyref

R = pyref.R_MOD
RS_TILE = 2048                 # keys per tile of the device radix sort (kRsTile in lookup.cu)
SMALL_SIZES = [1, 2, 31, 32, 33, 255, 256, 257, RS_TILE - 1, RS_TILE, RS_TILE + 1, 4 * RS_TILE + 1]


# ---- the reference ------------------------------------------------------------------------------------------------
def permute_reference(inp, tab):
    """Upstream permute_expression_pair over canonical integers: sort the input; count the table values in an ordered map;
    the first row of each distinct input value takes that value from the map; the leftover values, ascending, each go to the
    most recently pushed repeated row still unfilled. Raises ValueError when an input value is not in the table."""
    p_in = sorted(inp)
    leftover = Counter(tab)
    p_tab = [None] * len(inp)
    repeated = []
    for row, v in enumerate(p_in):
        if row > 0 and v == p_in[row - 1]:
            repeated.append(row)
            continue
        if leftover[v] == 0:
            raise ValueError("permute_expression_pair: %#x is not in the table (ConstraintSystemFailure)" % v)
        leftover[v] -= 1
        p_tab[row] = v
    for v in sorted(leftover):
        for _ in range(leftover[v]):
            p_tab[repeated.pop()] = v
    assert not repeated
    return p_in, p_tab


_MIX = np.array([0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0xD6E8FEB86659FD93], dtype=np.uint64)


def _same_rows(a, b):
    """whether the (n, 4) arrays hold the same rows with the same multiplicities. Both are sorted by a 64-bit mix of the
    limbs; equal results prove it. Only if they differ (which a collision of the mix could also cause) does a full
    lexicographic sort decide."""
    if np.array_equal(a[np.argsort((a * _MIX).sum(axis=1))], b[np.argsort((b * _MIX).sum(axis=1))]):
        return True
    return np.array_equal(a[np.lexsort(a.T)], b[np.lexsort(b.T)])


def check_lookup_definition(inp, tab, p_in, p_tab):
    """What the lookup argument needs of (p_in, p_tab), whatever algorithm made them: p_in is a permutation of inp, p_tab a
    permutation of tab, and on every row p_in[i] == p_tab[i] or (i > 0 and p_in[i] == p_in[i - 1]).
    Takes lists of integers, or (n, 4) uint64 limb arrays (Montgomery form is a bijection, so equality carries over)."""
    if isinstance(inp, np.ndarray):
        inp, tab, p_in, p_tab = [np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4) for a in (inp, tab, p_in, p_tab)]
        assert _same_rows(p_in, inp), "permuted input is not a permutation of the input"
        assert _same_rows(p_tab, tab), "permuted table is not a permutation of the table"
        ok = np.all(p_in == p_tab, axis=1)
        ok[1:] |= np.all(p_in[1:] == p_in[:-1], axis=1)
        bad = np.flatnonzero(~ok)
        assert bad.size == 0, "row %d: permuted input equals neither the permuted table nor the row above" % bad[0]
        return
    assert Counter(p_in) == Counter(inp), "permuted input is not a permutation of the input"
    assert Counter(p_tab) == Counter(tab), "permuted table is not a permutation of the table"
    for i in range(len(p_in)):
        assert p_in[i] == p_tab[i] or (i > 0 and p_in[i] == p_in[i - 1]), \
            "row %d: permuted input equals neither the permuted table nor the row above" % i


# ---- column shapes, each named for the branch of the device sort it reaches -----------------------------------------
def _random_fr(rng, count):
    r = random.Random(int(rng.integers(1 << 62)))
    return [r.randrange(R) for _ in range(count)]


def _distinct_random_fr(rng, count):
    vals = set()
    while len(vals) < count:
        vals.update(_random_fr(rng, count - len(vals)))
    return sorted(vals)


def _tiled(pool_size, n, rng):
    """table: the pool repeated to n rows (every value present when n >= pool_size); input: drawn from the table's values"""
    tab = np.arange(n) % pool_size
    return rng.integers(0, min(pool_size, n), n), tab


def shape_range(bits):
    """range table 0..2^bits (a halo2-lib range check): 1, 1, 2, 3, 3 counting-sort passes on limb 0 for bits = 5, 8, 12,
    19, 23 once n covers the range, none on limbs 1-3 -- odd and even pass counts"""
    def make(n, rng):
        pool = range(min(1 << bits, n))
        return (pool,) + _tiled(len(pool), n, rng)
    return make


def shape_top_and_low(n, rng):
    """a * 2^192 + b, a from three values, b random 64-bit: passes on limbs 0 and 3 only. Keys equal on the top limb must
    keep the order the limb-0 sort gave them (stability across limbs)."""
    tops = [1, 0x12345678, (R >> 192) - 1]
    d = max(1, min(n // 2, 1 << 14))
    lows = rng.integers(0, 1 << 64, d, dtype=np.uint64)
    pool = sorted(set((tops[int(t)] << 192) | int(b) for t, b in zip(rng.integers(0, 3, d), lows)))
    return (pool,) + _tiled(len(pool), n, rng)


def shape_top_only(n, rng):
    """k * 2^192 for small k: every byte of limbs 0-2 is the same, only the top limb is sorted (one pass)"""
    pool = [k << 192 for k in range(min(n, 200))]
    return (pool,) + _tiled(len(pool), n, rng)


def shape_negative(n, rng):
    """r - i for small i: the high bytes of the canonical form are constant, while the Montgomery form varies everywhere"""
    pool = sorted(R - i for i in range(1, min(n, 5000) + 1))
    return (pool,) + _tiled(len(pool), n, rng)


_BASE = (0x01020304 << 192) | 0x55
OUTLIERS = {"below": _BASE - 1,            # differs from the rest in the lowest byte of limb 0
            "above": _BASE + (1 << 200)}   # differs only in byte 1 of the top limb


def outlier_row(where, n):
    return {"first": 0, "last": n - 1, "mid": min(n - 1, n * 5 // 8 + 37)}[where]


def shape_one_outlier(where, value):
    """every key equal but one: one digit bucket holds n - 1 keys, so that digit must still be sorted"""
    def make(n, rng):
        pool = [_BASE, OUTLIERS[value]]
        idx = np.zeros(n, dtype=np.int64)
        idx[outlier_row(where, n)] = 1
        return pool, idx, idx.copy()
    return make


def shape_one_value(n, rng):
    """one input value on every row against a duplicate-free table: n - 1 repeated rows, every other table value a leftover"""
    pool = _distinct_random_fr(rng, n)
    return pool, np.full(n, int(rng.integers(0, n))), rng.permutation(n)


def shape_permutation(n, rng):
    """input a permutation of a duplicate-free table: no repeated rows and no leftovers"""
    pool = _distinct_random_fr(rng, n)
    return pool, rng.permutation(n), rng.permutation(n)


def spectre_table_bits(n):
    """the range table an aggregation circuit with 2^K - 7 usable rows looks up: 2^min(19, K - 1) values"""
    return max(0, min(19, (n + 7).bit_length() - 2))


def shape_spectre(table_bits=None):
    """Spectre's lookup column: a range table padded with zeros to the usable rows, and an input that is 0 on ~70 % of
    the rows and a table value elsewhere. The value 0 has ~n leftovers."""
    def make(n, rng):
        bits = spectre_table_bits(n) if table_bits is None else table_bits
        pool = range(min(1 << bits, n))
        tab = np.zeros(n, dtype=np.int64)
        tab[:len(pool)] = np.arange(len(pool))
        inp = rng.integers(0, len(pool), n)
        inp[rng.random(n) < 0.7] = 0
        return pool, inp, tab
    return make


def shape_theta(n, rng):
    """random 256-bit values each repeated many times (a theta-compressed multi-column lookup): 8 passes on every limb"""
    pool = _random_fr(rng, max(1, n // 64))
    return (pool,) + _tiled(len(pool), n, rng)


SHAPES = {
    **{"range%d" % b: shape_range(b) for b in (5, 8, 12, 19, 23)},
    "top_and_low": shape_top_and_low,
    "top_only": shape_top_only,
    "negative": shape_negative,
    **{"outlier_%s_%s" % (w, v): shape_one_outlier(w, v) for w in ("first", "mid", "last") for v in OUTLIERS},
    "one_value": shape_one_value,
    "permutation": shape_permutation,
    "spectre": shape_spectre(),
    "theta": shape_theta,
}


def make_shape(name, n, seed):
    return SHAPES[name](n, np.random.default_rng(seed))


def mont_pool(orc, pool):
    """Montgomery limbs of the pool's values; a range 0..m is built by the oracle's repeated addition"""
    if isinstance(pool, range) and pool.start == 0 and pool.step == 1:
        return orc.fr_seq(len(pool))
    return orc.fr(list(pool))


# ---- missing table values ----------------------------------------------------------------------------------------------
MISSING = ("below", "between", "above")
PLACEMENTS = ("first_row", "last_row", "only_value")


def shape_missing(where, placement, n, seed):
    """a valid column with one value that is not in the table: below the table's minimum, between two table values, or
    above its maximum (the device's binary search runs off the end); on the input's first row, its last row, or on every
    row. Table values are 10, 20, ..."""
    rng = np.random.default_rng(seed)
    d = max(2, min(n, 300))
    pool = [10 * (i + 1) for i in range(d)] + [{"below": 3, "between": 15, "above": R - 1}[where]]
    tab = np.arange(n) % min(d, n)
    inp = rng.integers(0, min(d, n), n)
    rows = {"first_row": [0], "last_row": [n - 1], "only_value": slice(None)}[placement]
    inp[rows] = d
    return pool, inp, tab


# ---- the restatement against the oracle ----------------------------------------------------------------------------
def _ints(pool, idx):
    return [pool[int(i)] for i in idx]


@pytest.mark.parametrize("n", SMALL_SIZES + [(1 << 14) - 7])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_reference_matches_oracle(orc, shape, n):
    pool, ii, ti = make_shape(shape, n, seed=n)
    inp, tab = _ints(pool, ii), _ints(pool, ti)
    p_in, p_tab = permute_reference(inp, tab)
    check_lookup_definition(inp, tab, p_in, p_tab)
    mp = mont_pool(orc, pool)
    o_in, o_tab = orc.permute_expression_pair(mp[ii], mp[ti])
    assert orc.fr_ints(o_in) == p_in
    assert orc.fr_ints(o_tab) == p_tab
    check_lookup_definition(mp[ii], mp[ti], o_in, o_tab)


@pytest.mark.parametrize("n", [2, 33, RS_TILE + 1])
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("where", MISSING)
def test_reference_and_oracle_reject_missing_value(orc, where, placement, n):
    pool, ii, ti = shape_missing(where, placement, n, seed=n)
    with pytest.raises(ValueError, match="ConstraintSystemFailure"):
        permute_reference(_ints(pool, ii), _ints(pool, ti))
    mp = mont_pool(orc, pool)
    with pytest.raises(ValueError, match="ConstraintSystemFailure"):
        orc.permute_expression_pair(mp[ii], mp[ti])


def test_reference_leftover_order():
    """a hand-checked case: input 1 1 1 2 2 against table 1 2 3 3 4. Repeated rows 1, 2, 4 take the leftovers 3, 3, 4
    from the last repeated row backwards."""
    p_in, p_tab = permute_reference([2, 1, 2, 1, 1], [3, 1, 4, 2, 3])
    assert p_in == [1, 1, 1, 2, 2]
    assert p_tab == [1, 4, 3, 2, 3]


@pytest.mark.parametrize("as_limbs", [False, True])
def test_check_lookup_definition_rejects(orc, as_limbs):
    """the checker fails on each way a permuted pair can be wrong"""
    inp, tab = [5, 1, 5, 7, 5, 1], [1, 9, 5, 7, 1, 8]
    p_in, p_tab = permute_reference(inp, tab)
    conv = (lambda x: orc.fr(x)) if as_limbs else (lambda x: list(x))
    check_lookup_definition(conv(inp), conv(tab), conv(p_in), conv(p_tab))
    swapped = list(p_tab); swapped[0], swapped[1] = swapped[1], swapped[0]        # still a permutation, row 0 breaks
    changed = list(p_tab); changed[2] = 9                                         # not a permutation of the table
    unsorted_in = list(p_in); unsorted_in[0], unsorted_in[3] = unsorted_in[3], unsorted_in[0]
    for a, b in ((p_in, swapped), (p_in, changed), (unsorted_in, p_tab), ([1] * 6, p_tab)):
        with pytest.raises(AssertionError):
            check_lookup_definition(conv(inp), conv(tab), conv(a), conv(b))
