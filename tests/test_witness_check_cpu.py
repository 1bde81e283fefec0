"""The witness check (plonk.check_witness, halo2's MockProver::verify) on the CPU: the device bodies of witness.cu run serially
(tests/hostemu/witness.cpp, with and without the PTX emulation), and check_witness driven by a CPU engine built on them equals
an independent pure-Python MockProver on clean witnesses and on injected faults."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from spectre_b200 import circuits, plonk
from spectre_b200.plonk import R_MOD, WitnessFailure
from tests.plonk_oracle_engine import OracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTANCES = [3, 1, 4]


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _build(tmp_path_factory, name, flags):
    so = str(tmp_path_factory.mktemp("hostemu_witness") / name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, os.path.join(ROOT, "tests", "hostemu", "witness.cpp")])
    lib = ctypes.CDLL(so)
    lib.he_compact.restype = ctypes.c_uint64
    return lib


@pytest.fixture(scope="module")
def he_host(tmp_path_factory):
    return _build(tmp_path_factory, "libhostemu_witness.so", [])


@pytest.fixture(scope="module", params=["host64", "ptx"])
def he(request, tmp_path_factory, he_host):
    return he_host if request.param == "host64" else _build(tmp_path_factory, "libhostemu_witness_ptx.so", ["-DSPB_EMULATE_PTX"])


def _ptrs(arrs):
    return (ctypes.c_void_p * max(1, len(arrs)))(*[a.ctypes.data for a in arrs])


def compact(he, flags, lo, hi, cap):
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    out = np.zeros(max(cap, 1), dtype=np.uint32)
    total = he.he_compact(_p(flags), ctypes.c_uint64(lo), ctypes.c_uint64(hi), ctypes.c_uint64(cap), _p(out))
    return [int(r) for r in out[:min(cap, total)]], int(total)


# ---- a CPU engine whose witness-check methods run the device bodies -------------------------------------------------------
class WitnessOracleEngine(OracleEngine):
    def __init__(self, he, k, j):
        super().__init__(k, j)
        self.he = he

    def nonzero_rows(self, values, lo, hi, cap):
        return compact(self.he, values.a[lo:hi].any(axis=1), lo, hi, cap)

    def lookup_missing_rows(self, ci, ct, usable, cap):
        missing = np.zeros(usable, dtype=np.uint8)
        self.he.he_lookup_missing(_p(np.ascontiguousarray(ci.a[:usable])), _p(np.ascontiguousarray(ct.a[:usable])), ctypes.c_uint64(usable), _p(missing))
        return compact(self.he, missing, 0, usable, cap)

    def copy_mismatches(self, values, sigma, usable, cap):
        vals, sig = [np.ascontiguousarray(b.a) for b in values], [np.ascontiguousarray(b.a) for b in sigma]
        out = []
        for c in range(len(vals)):
            rc, cols, rows = np.zeros(usable, np.int32), np.zeros(usable, np.uint32), np.zeros(usable, np.uint64)
            self.he.he_copy_check(ctypes.c_uint32(self.k), _ptrs(vals), _ptrs(sig), ctypes.c_uint32(len(vals)), ctypes.c_uint32(c), ctypes.c_uint64(usable),
                                  _p(rc), _p(cols), _p(rows))
            bad = np.nonzero(rc == 2)[0]
            if bad.size:
                raise ValueError("sigma of permutation column %d, row %d labels no usable cell" % (c, bad[0]))
            rs, total = compact(self.he, rc == 1, 0, usable, cap)
            out.append((total, [(r, int(cols[r]), int(rows[r])) for r in rs]))
        return out


# ---- the independent MockProver: Python ints, straight from the semantics --------------------------------------------------
def _ints(col):
    return [plonk.fr_int(r) for r in col]


def mock_prover(pk, instances, advice_columns, max_rows=16):
    cs, k, n, u = pk.cs, pk.k, pk.n, pk.usable_rows
    E = OracleEngine(k, 3)
    cols = {"fixed": [_ints(E.download(b)) for b in pk.fixed_values], "advice": [_ints(a) for a in advice_columns],
            "instance": [[v % R_MOD for v in col] + [0] * (n - len(col)) for col in instances]}

    def ev(e, i):
        t = e[0]
        if t == "const": return e[1]
        if t in cols: return cols[t][e[1]][(i + e[2]) % n]
        if t == "neg": return -ev(e[1], i) % R_MOD
        if t == "sum": return (ev(e[1], i) + ev(e[2], i)) % R_MOD
        if t == "prod": return ev(e[1], i) * ev(e[2], i) % R_MOD
        return ev(e[1], i) * e[2] % R_MOD

    out = []

    def report(kind, index, rows, mapped=None):
        if rows:
            out.append(WitnessFailure(kind, index, rows[:max_rows], len(rows), mapped[:max_rows] if mapped is not None else None))
    for g, gate in enumerate(cs.gates):
        report("gate", g, [i for i in range(u) if ev(gate, i)])
    for li, (ins, tbs) in enumerate(cs.lookups):
        table = {tuple(ev(e, j) for e in tbs) for j in range(u)}
        report("lookup", li, [i for i in range(u) if tuple(ev(e, i) for e in ins) not in table])
    w = plonk.omega_of(k)
    labels = {plonk.DELTA ** c * pow(w, i, R_MOD) % R_MOD: (c, i) for c in range(len(cs.permutation)) for i in range(n)}
    values = [cols[kind][c] for kind, c in cs.permutation]
    for c, s in enumerate(pk.sigma_values):
        sig = _ints(E.download(s))
        bad = [(i, labels[sig[i]]) for i in range(u) if values[c][i] != values[labels[sig[i]][0]][labels[sig[i]][1]]]
        report("copy", c, [i for i, _ in bad], [m for _, m in bad])
    return out


# ---- the bodies ---------------------------------------------------------------------------------------------------------
class _Perm:
    def __init__(self, cols):
        self.permutation = [("advice", c) for c in range(cols)]


@pytest.mark.parametrize("k,cols", [(3, 1), (4, 2), (5, 21), (6, 3), (7, 5), (8, 1), (9, 7), (10, 2), (11, 4), (12, 21)])
def test_sigma_decode_recovers_every_cell(he, orc, k, cols):
    """every sigma entry of a key from build_sigma (random copies, so non-trivial cycles) decodes to the cell Python's pow labels,
    the maximum usable row u - 1 among them; a corrupted entry decodes to no cell"""
    n = 1 << k
    E = OracleEngine(k, 3)
    rng = random.Random(1000 * k + cols)
    u = n - 7
    copies = [((rng.randrange(cols), rng.randrange(u)), (rng.randrange(cols), rng.randrange(u))) for _ in range(n // 4)]
    copies.append(((cols - 1, u - 1), (0, u - 1)))                  # the last usable row on a cycle
    sigma = plonk.build_sigma(E, _Perm(cols), k, copies)
    w = plonk.omega_of(k)
    labels = {plonk.DELTA ** c * pow(w, i, R_MOD) % R_MOD: (c, i) for c in range(cols) for i in range(n)}
    for c, s in enumerate(sigma):
        a = np.ascontiguousarray(s.a)
        got_c, got_r, ok = np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint8)
        he.he_sigma_decode(_p(a), ctypes.c_uint64(n), ctypes.c_uint32(k), ctypes.c_uint32(cols), _p(got_c), _p(got_r), _p(ok))
        assert ok.all()
        assert [(int(x), int(y)) for x, y in zip(got_c, got_r)] == [labels[v] for v in _ints(a)], "column %d" % c
    bad = np.stack([plonk.fr_mont(rng.randrange(R_MOD)), plonk.fr_mont(plonk.DELTA ** cols % R_MOD)])   # random; column C (one past the last)
    got_c, got_r, ok = np.zeros(2, np.uint32), np.zeros(2, np.uint64), np.ones(2, np.uint8)
    he.he_sigma_decode(_p(bad), ctypes.c_uint64(2), ctypes.c_uint32(k), ctypes.c_uint32(cols), _p(got_c), _p(got_r), _p(ok))
    assert not ok.any()


def test_copy_check_row_flags_mismatches_and_malformed_entries(he, orc):
    k, cols = 6, 3
    n = 1 << k
    u = n - 7
    E = OracleEngine(k, 3)
    sigma = [np.ascontiguousarray(s.a) for s in plonk.build_sigma(E, _Perm(cols), k, [((0, 5), (2, 9)), ((1, u - 1), (0, 0))])]
    values = [np.ascontiguousarray(orc.fr_random_chacha(n, 0x5eed2000 + c)) for c in range(cols)]
    values[2][9] = values[0][5]
    values[0][0] = values[1][u - 1]
    values[1][u - 1] = plonk.fr_mont(plonk.fr_int(values[1][u - 1]) + 1)             # breaks (1, u-1) -> (0, 0) and (0, 0) -> (1, u-1)

    def run(c):
        rc, cc, rr = np.zeros(u, np.int32), np.zeros(u, np.uint32), np.zeros(u, np.uint64)
        he.he_copy_check(ctypes.c_uint32(k), _ptrs(values), _ptrs(sigma), ctypes.c_uint32(cols), ctypes.c_uint32(c), ctypes.c_uint64(u), _p(rc), _p(cc), _p(rr))
        return rc, cc, rr
    rc, cc, rr = run(0)
    assert list(np.nonzero(rc)[0]) == [0] and rc[0] == 1 and (cc[0], rr[0]) == (1, u - 1)
    assert rc[5] == 0 and (cc[5], rr[5]) == (2, 9)
    rc, cc, rr = run(1)
    assert list(np.nonzero(rc)[0]) == [u - 1] and (cc[u - 1], rr[u - 1]) == (0, 0)
    sigma[2][3] = plonk.fr_mont(plonk.DELTA ** 1 * pow(plonk.omega_of(k), n - 1, R_MOD) % R_MOD)   # labels a blinding row
    rc, _, _ = run(2)
    assert list(np.nonzero(rc)[0]) == [3] and rc[3] == 2


@pytest.mark.parametrize("lo,hi,cap", [(0, 1000, 16), (5, 517, 4), (0, 256, 300), (3, 4, 1), (0, 70000, 16)])
def test_compaction_matches_python(he, lo, hi, cap):
    rng = np.random.default_rng(lo * 7 + hi + cap)
    m = hi - lo
    last = np.zeros(m, np.uint8); last[-1] = 1
    few = np.zeros(m, np.uint8); few[rng.choice(m, size=min(m, cap + 3), replace=False)] = 1   # more than cap when m allows
    for flags in (np.zeros(m, np.uint8), np.ones(m, np.uint8), last, few, (rng.random(m) < 0.01).astype(np.uint8)):
        want = [lo + i for i in np.nonzero(flags)[0]]
        assert compact(he, flags, lo, hi, cap) == ([int(r) for r in want[:cap]], len(want))


def test_lookup_membership_matches_python(he):
    rng = random.Random(7)
    u = 600
    table_vals = [rng.randrange(R_MOD) for _ in range(40)] + [0, R_MOD - 1]
    table = [table_vals[rng.randrange(len(table_vals))] for _ in range(u)]
    inputs = [table_vals[rng.randrange(len(table_vals))] if rng.random() < 0.9 else rng.randrange(R_MOD) for _ in range(u)]
    inputs[-1] = R_MOD - 2
    missing = np.zeros(u, np.uint8)
    he.he_lookup_missing(_p(plonk.fr_mont_rows(inputs)), _p(plonk.fr_mont_rows(table)), ctypes.c_uint64(u), _p(missing))
    assert [bool(m) for m in missing] == [v not in set(table) for v in inputs]
    assert missing[-1]


# ---- check_witness against the MockProver -------------------------------------------------------------------------------
def _case(shape, k):
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, INSTANCES, lookup_bits=3, groups=30)
        return cs, fixed, [adv], copies
    if shape == "wide":
        cs = circuits.wide_shape(3)
        fixed, adv, copies = circuits.wide_witness(cs, k, INSTANCES, lookup_bits=3, groups=20)
        return cs, fixed, adv, copies
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, INSTANCES, lookup_bits=4, groups=20, num_gate_advice=3, num_lookup_advice=2)
    return cs, fixed, adv, copies


def _key(he, shape, k):
    cs, fixed, adv, copies = _case(shape, k)
    E = WitnessOracleEngine(he, k, cs.degree())
    return E, plonk.keygen(E, cs, k, fixed, copies), adv


@pytest.mark.parametrize("shape,k", [("aggregation", 7), ("wide", 7), ("halo2lib", 8)])
def test_clean_witness_has_no_failures(he_host, orc, shape, k):
    E, pk, adv = _key(he_host, shape, k)
    assert plonk.check_witness(E, pk, [INSTANCES], adv) == []
    assert mock_prover(pk, [INSTANCES], adv) == []


def _bump(col, row, by=1):
    col[row] = plonk.fr_mont(plonk.fr_int(col[row]) + by)


def faults():
    """(name, shape, k, instances, mutate(advice columns), max_rows)"""
    def rot3(adv):                                              # d of group 5, read by the gate at row 20 through rotation 3
        _bump(adv[0], 23)

    def tuple_not_in_table(adv):                                # wide lookup: (a, a^2 + 1) rows; column 1 gets another entry's
        r = 4 * 6                                               # second coordinate, so each value is in its table column
        a = plonk.fr_int(adv[0][r])
        other = (a + 1) % 8
        adv[1][r] = plonk.fr_mont(other * other + 1)
        b, c = plonk.fr_int(adv[1][r + 1]), plonk.fr_int(adv[1][r + 2])
        adv[1][r + 3] = plonk.fr_mont(other * other + 1 + b * c)   # the gate of column 1 still holds

    def across_sets(adv):                                       # advice 2 row 1 (set 0) is copied to the constants cell (set 1)
        _bump(adv[2], 1)

    def many(adv):                                              # every group's d: more failures of the gate than max_rows
        for g in range(29):                                     # the 29 groups that fit in the 121 usable rows of k = 7
            _bump(adv[0], 4 * g + 3, 5)
    return [("rotation3", "aggregation", 7, INSTANCES, rot3, 16),
            ("tuple", "wide", 7, INSTANCES, tuple_not_in_table, 16),
            ("across_sets", "wide", 7, INSTANCES, across_sets, 16),
            ("public_input", "halo2lib", 8, [3, 9, 4], lambda adv: None, 16),
            ("many", "aggregation", 7, INSTANCES, many, 4)]


@pytest.mark.parametrize("name,shape,k,instances,mutate,max_rows", faults(), ids=[f[0] for f in faults()])
def test_injected_faults_match_the_mock_prover(he_host, orc, name, shape, k, instances, mutate, max_rows):
    E, pk, adv = _key(he_host, shape, k)
    adv = [a.copy() for a in adv]
    mutate(adv)
    want = mock_prover(pk, [instances], adv, max_rows)
    got = plonk.check_witness(E, pk, [instances], adv, theta=0x5eed + k, max_rows=max_rows)
    assert got == want
    assert got
    kinds = {f.kind for f in got}
    expect = {"rotation3": "gate", "tuple": "lookup", "across_sets": "copy", "public_input": "copy", "many": "gate"}[name]
    assert expect in kinds, got
    if name == "tuple":
        assert got == [WitnessFailure("lookup", 0, [24], 1)]
    if name == "across_sets":
        assert any(f.kind == "copy" and f.index == 3 and f.mapped == [(2, 1)] for f in got), got
    if name == "many":
        gate = [f for f in got if f.kind == "gate"][0]
        assert gate.total == 29 and gate.rows == [0, 4, 8, 12]


def test_instances_are_laid_out_as_create_proof_lays_them_out(he_host, orc):
    E, pk, adv = _key(he_host, "aggregation", 6)
    with pytest.raises(ValueError, match="InstanceTooLarge"):
        plonk.check_witness(E, pk, [[1] * (pk.usable_rows + 1)], adv)
    with pytest.raises(ValueError, match="InvalidInstances"):
        plonk.check_witness(E, pk, [], adv)
