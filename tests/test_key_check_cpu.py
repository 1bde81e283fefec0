"""The proving-key check (plonk.check_pk and the checked plonk.read_pk) on the CPU: the device bodies of the key check run
serially (tests/hostemu/key_check.cpp, with and without the PTX emulation), and check_pk driven by a CPU engine built on them
equals an independent pure-Python audit of the key on injected faults."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from spectre_b200 import circuits, halo2, plonk
from spectre_b200.plonk import DELTA, P_MOD, R_MOD, ZETA, KeyFailure
from tests.test_witness_check_cpu import WitnessOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTANCES = [3, 1, 4]
OTHER_TAU = 0x7a0f3e5d


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _build(tmp_path_factory, name, flags):
    so = str(tmp_path_factory.mktemp("hostemu_key_check") / name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, os.path.join(ROOT, "tests", "hostemu", "key_check.cpp")])
    lib = ctypes.CDLL(so)
    lib.he_compact.restype = ctypes.c_uint64
    lib.he_fr_first_noncanonical.restype = ctypes.c_uint64
    return lib


@pytest.fixture(scope="module")
def he_host(tmp_path_factory):
    return _build(tmp_path_factory, "libhostemu_key_check.so", [])


@pytest.fixture(scope="module", params=["host64", "ptx"])
def he(request, tmp_path_factory, he_host):
    return he_host if request.param == "host64" else _build(tmp_path_factory, "libhostemu_key_check_ptx.so", ["-DSPB_EMULATE_PTX"])


def he_sigma_check(he, k, sigma, usable, cap):
    """the CPU twin of Backend.sigma_check_dev: sigma = list of (n, 4) arrays"""
    sig = [np.ascontiguousarray(s, dtype=np.uint64) for s in sigma]
    m = len(sig)
    ptrs = (ctypes.c_void_p * max(1, m))(*[s.ctypes.data for s in sig])
    rows, totals = np.zeros(max(3 * m * cap, 1), np.uint32), np.zeros(max(3 * m, 1), np.uint64)
    he.he_sigma_check(ctypes.c_uint32(k), ptrs, ctypes.c_uint32(m), ctypes.c_uint64(usable), ctypes.c_uint32(cap), _p(rows), _p(totals))
    return [[(int(totals[3 * c + q]), [int(r) for r in rows[(3 * c + q) * cap:(3 * c + q) * cap + min(cap, int(totals[3 * c + q]))]]) for q in range(3)]
            for c in range(m)]


# ---- a CPU engine whose key-check methods run the device bodies --------------------------------------------------------------
class KeyCheckOracleEngine(WitnessOracleEngine):
    """tau: None for the oracle's seed-0 SRS; otherwise commit_lagrange is made under an SRS with that secret"""

    def __init__(self, he, k, j, tau=None):
        super().__init__(he, k, j)
        self.tau = tau

    def commit(self, basis, bufs, n):
        if self.tau is None:
            return super().commit(basis, bufs, n)
        from oracle import oracle as orc
        out = []
        for b in bufs:
            coeffs = b.a[:n] if basis == halo2.BASIS_G else self.dom.lagrange_to_coeff(np.ascontiguousarray(b.a[:n]))
            s = orc.eval_polynomial(coeffs, plonk.fr_mont(self.tau))
            out.append(tuple(orc.affine_ints(orc.g1_to_affine(orc.g1_mul(orc.g1_generator(), s)))[0]))
        return out

    def first_noncanonical(self, b, rows):
        return int(self.he.he_fr_first_noncanonical(_p(np.ascontiguousarray(b.a[:rows])), ctypes.c_uint64(rows)))

    def sigma_check(self, sigma, usable, cap):
        return he_sigma_check(self.he, self.k, [s.a for s in sigma], usable, cap)

    def vec_axpy(self, y, alpha, x, n):
        a = plonk.fr_int(alpha)
        y.a[:n] = plonk.fr_mont_rows([(plonk.fr_int(u) + a * plonk.fr_int(v)) % R_MOD for u, v in zip(y.a[:n], x.a[:n])])


# ---- the independent audit: Python ints, straight from the definitions ----------------------------------------------------
def _ints(a):
    return [plonk.fr_int(r) for r in a]


def _lagrange_eval(vals, x, k):
    """sum_i vals[i] L_i(x), L_i(x) = omega^i (x^n - 1) / (n (x - omega^i)), for x outside the 2^k-th roots of unity"""
    n, w = 1 << k, plonk.omega_of(k)
    zn = (pow(x, n, R_MOD) - 1) * pow(n, -1, R_MOD) % R_MOD
    acc, wi = 0, 1
    for v in vals:
        if v:
            acc += v * wi * pow(x - wi, -1, R_MOD)
        wi = wi * w % R_MOD
    return acc * zn % R_MOD


def _horner(coeffs, x):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % R_MOD
    return acc


def _labels(k, cols):
    w = plonk.omega_of(k)
    return {DELTA ** c * pow(w, i, R_MOD) % R_MOD: (c, i) for c in range(cols) for i in range(1 << k)}


def sigma_audit(k, sigma_rows, usable, max_rows=16):
    """sigma_rows: per column a list of raw (n, 4) limb rows -> the three kinds per column, as spb_sigma_check_dev reports them"""
    n, cols = 1 << k, len(sigma_rows)
    labels = _labels(k, cols)
    own = {v: key for key, v in labels.items()}
    hit = set()
    out = []
    for c, col in enumerate(sigma_rows):
        kinds = [[], [], []]
        for i, raw in enumerate(col):
            r = int(raw[0]) | int(raw[1]) << 64 | int(raw[2]) << 128 | int(raw[3]) << 192
            target = labels.get(plonk.fr_int(raw)) if r < R_MOD else None
            if target is not None:
                hit.add(target)
            if i < usable and (target is None or target[1] >= usable):
                kinds[0].append(i)
            if i >= usable and target != (c, i):
                kinds[1].append(i)
        out.append(kinds)
    for c in range(cols):
        out[c][2] = [i for i in range(n) if (c, i) not in hit]
    assert len(own) == len(labels)
    return [[(len(rs), rs[:max_rows]) for rs in kinds] for kinds in out]


def key_audit(E, pk, tau, max_rows=16):
    """check_pk restated: commitments by the Lagrange formula at tau, NTTs and coset NTTs as evaluations, sigma from its
    definition; the stored key is read through the engine's download only"""
    k, n, u = pk.k, pk.n, pk.usable_rows
    ext_k = E.extended_k
    w, ext_w = plonk.omega_of(k), pow(plonk.ROOT_OF_UNITY, 1 << (28 - ext_k), R_MOD)
    from oracle import oracle as orc
    out = []

    def rows_of(kind, index, bad):
        if bad:
            out.append(KeyFailure(kind, index, bad[:max_rows], len(bad)))
    fv, sv = [_ints(E.download(b)) for b in pk.fixed_values], [_ints(E.download(b)) for b in pk.sigma_values]
    fp, sp = [_ints(E.download(b)) for b in pk.fixed_polys], [_ints(E.download(b)) for b in pk.sigma_polys]
    for kind, vals, vk in (("fixed_commitment", fv, pk.fixed_commitments), ("sigma_commitment", sv, pk.sigma_commitments)):
        for i, (v, pt) in enumerate(zip(vals, vk)):
            s = _lagrange_eval(v, tau, k)
            want = tuple(orc.affine_ints(orc.g1_to_affine(orc.g1_mul(orc.g1_generator(), plonk.fr_mont(s))))[0])
            if want != tuple(pt):
                out.append(KeyFailure(kind, i, None, 1))
    for kind, vals, coeffs in (("fixed_poly", fv, fp), ("sigma_poly", sv, sp)):
        for i, (v, p) in enumerate(zip(vals, coeffs)):
            rows_of(kind, i, [r for r in range(n) if _horner(p, pow(w, r, R_MOD)) != v[r]])
    if not pk.lean:
        pts = [ZETA * pow(ext_w, j, R_MOD) % R_MOD for j in range(1 << ext_k)]
        for kind, coeffs, cosets in (("fixed_coset", fp, pk.fixed_cosets), ("sigma_coset", sp, pk.sigma_cosets)):
            for i, (p, c) in enumerate(zip(coeffs, cosets)):
                cv = _ints(E.download(c))
                rows_of(kind, i, [j for j, x in enumerate(pts) if _horner(p, x) != cv[j]])
        ldefs = [[1] + [0] * (n - 1), [0] * u + [1] + [0] * (n - u - 1), [1] * u + [0] * (n - u)]
        for i, (vals, c) in enumerate(zip(ldefs, (pk.l0, pk.l_last, pk.l_active))):
            cv = _ints(E.download(c))
            rows_of("l_coset", i, [j for j, x in enumerate(pts) if _lagrange_eval(vals, x, k) != cv[j]])
    if pk.sigma_values:
        rep = sigma_audit(k, [E.download(b) for b in pk.sigma_values], u, max_rows)
        for q, kind in enumerate(("sigma_label", "sigma_blinding", "sigma_unlabelled")):
            for c, kinds in enumerate(rep):
                total, rows = kinds[q]
                if total:
                    out.append(KeyFailure(kind, c, rows, total))
    return out


# ---- the bodies ---------------------------------------------------------------------------------------------------------
def _raw(v):
    return np.array([(v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)


def test_canonical_test_matches_python_integers(he):
    rng = random.Random(11)
    vals = [0, 1, R_MOD - 1, R_MOD, R_MOD + 1, (1 << 256) - 1, (1 << 255), R_MOD - (1 << 64)] + [rng.getrandbits(256) for _ in range(200)]
    vals += [rng.randrange(R_MOD) for _ in range(50)]
    arr = np.stack([_raw(v) for v in vals])
    for i, v in enumerate(vals):
        got = int(he.he_fr_first_noncanonical(_p(np.ascontiguousarray(arr[i:i + 1])), ctypes.c_uint64(1)))
        assert got == (0 if v >= R_MOD else 1), hex(v)
    first = next(i for i, v in enumerate(vals) if v >= R_MOD)
    assert int(he.he_fr_first_noncanonical(_p(arr), ctypes.c_uint64(len(vals)))) == first
    ok = np.stack([_raw(rng.randrange(R_MOD)) for _ in range(64)])
    assert int(he.he_fr_first_noncanonical(_p(ok), ctypes.c_uint64(64))) == 64
    assert int(he.he_fr_first_noncanonical(_p(ok), ctypes.c_uint64(0))) == 0


class _Perm:
    def __init__(self, cols):
        self.permutation = [("advice", c) for c in range(cols)]


def faulty_sigma(E, k, cols, seed):
    """a sigma from build_sigma with random copies, then one entry of each malformed kind"""
    n = 1 << k
    u = n - 7
    rng = random.Random(seed)
    copies = [((rng.randrange(cols), rng.randrange(u)), (rng.randrange(cols), rng.randrange(u))) for _ in range(n // 4)]
    sigma = [E.download(s) for s in plonk.build_sigma(E, _Perm(cols), k, copies)]
    w = plonk.omega_of(k)
    lab = lambda c, i: plonk.fr_mont(DELTA ** c * pow(w, i, R_MOD) % R_MOD)
    sigma[rng.randrange(cols)][rng.randrange(u)] = plonk.fr_mont(rng.randrange(R_MOD))         # labels nothing
    sigma[rng.randrange(cols)][rng.randrange(u)] = lab(rng.randrange(cols), u + 1)             # labels a blinding row
    sigma[rng.randrange(cols)][u + 2] = lab(rng.randrange(cols), rng.randrange(u))             # a blinding row moved
    sigma[cols - 1][0] = lab(cols, 3)                                                         # column C, one past the last
    sigma[0][u - 1] = _raw(R_MOD)                                                            # not canonical
    return sigma, u


@pytest.mark.parametrize("k,cols", [(3, 1), (4, 2), (5, 21), (6, 3), (7, 5), (8, 1), (9, 7), (10, 2), (11, 4), (12, 21)])
def test_sigma_check_matches_python(he, orc, k, cols):
    E = KeyCheckOracleEngine(he, k, 3)
    sigma, u = faulty_sigma(E, k, cols, 77 * k + cols)
    for cap in (16, 2):
        assert he_sigma_check(he, k, sigma, u, cap) == sigma_audit(k, sigma, u, cap)
    clean = [E.download(s) for s in plonk.build_sigma(E, _Perm(cols), k, [((0, u // 2), (cols - 1, u - 1))])]
    assert he_sigma_check(he, k, clean, u, 16) == [[(0, [])] * 3] * cols
    assert he_sigma_check(he, k, clean, 1 << k, 16) == [[(0, [])] * 3] * cols          # no blinding rows: the same
    rep = he_sigma_check(he, k, clean, 0, 16)                                            # no usable rows: every copy is a fault
    assert rep == sigma_audit(k, clean, 0, 16)


# ---- check_pk against the audit -----------------------------------------------------------------------------------------
def key_case(k=7):
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, INSTANCES, lookup_bits=3, groups=30)
    return cs, fixed, copies


def _bump(E, b, row, by=1):
    E.write_rows(b, row, plonk.fr_mont(plonk.fr_int(E.read_rows(b, row, 1)[0]) + by).reshape(1, 4))


def _label(k, c, i):
    return plonk.fr_mont(DELTA ** c * pow(plonk.omega_of(k), i, R_MOD) % R_MOD).reshape(1, 4)


def key_faults():
    """(name, mutate(E, pk), max_rows, needs cosets)"""
    def fixed_value(E, pk): _bump(E, pk.fixed_values[1], 37)
    def fixed_coeff(E, pk): _bump(E, pk.fixed_polys[2], 5)
    def fixed_coset(E, pk): _bump(E, pk.fixed_cosets[0], 300)

    def sigma_swap(E, pk):
        s = pk.sigma_values[1]
        a, b = E.read_rows(s, 10, 1), E.read_rows(s, 20, 1)
        E.write_rows(s, 10, b); E.write_rows(s, 20, a)

    def sigma_relabel(E, pk): E.write_rows(pk.sigma_values[0], 11, _label(pk.k, 2, 50))
    def sigma_random(E, pk): E.write_rows(pk.sigma_values[2], 33, plonk.fr_mont(random.Random(5).randrange(R_MOD)).reshape(1, 4))
    def sigma_blinding(E, pk): E.write_rows(pk.sigma_values[1], pk.n - 3, _label(pk.k, 0, 7))

    def many(E, pk):
        for r in range(0, 40, 2):
            _bump(E, pk.fixed_values[3], r, 3)
    return [("clean", lambda E, pk: None, 16, False), ("fixed_value", fixed_value, 16, False), ("fixed_coeff", fixed_coeff, 16, False),
            ("fixed_coset", fixed_coset, 16, True), ("sigma_swap", sigma_swap, 16, False), ("sigma_relabel", sigma_relabel, 16, False),
            ("sigma_random", sigma_random, 16, False), ("sigma_blinding", sigma_blinding, 16, False), ("many", many, 4, False)]


def expected_shape(name, got, pk):
    """what each fault must show, beyond equality with the audit"""
    kinds = [(f.kind, f.index) for f in got]
    if name == "clean":
        assert got == []
    if name == "fixed_value":
        assert got == [KeyFailure("fixed_commitment", 1, None, 1), KeyFailure("fixed_poly", 1, [37], 1)]
    if name == "fixed_coeff":
        assert KeyFailure("fixed_poly", 2, list(range(16)), pk.n) in got
    if name == "fixed_coset":
        assert got == [KeyFailure("fixed_coset", 0, [300], 1)]
    if name == "sigma_swap":
        assert got == [KeyFailure("sigma_commitment", 1, None, 1), KeyFailure("sigma_poly", 1, [10, 20], 2)]
    if name == "sigma_relabel":
        assert kinds == [("sigma_commitment", 0), ("sigma_poly", 0), ("sigma_unlabelled", kinds[-1][1])] and got[-1].total == 1
    if name == "sigma_random":
        assert kinds[:2] == [("sigma_commitment", 2), ("sigma_poly", 2)]
        assert KeyFailure("sigma_label", 2, [33], 1) in got and [f.kind for f in got].count("sigma_unlabelled") == 1
    if name == "sigma_blinding":
        assert KeyFailure("sigma_blinding", 1, [pk.n - 3], 1) in got and KeyFailure("sigma_unlabelled", 1, [pk.n - 3], 1) in got
    if name == "many":
        assert KeyFailure("fixed_poly", 3, [0, 2, 4, 6], 20) in got


@pytest.mark.parametrize("name,mutate,max_rows,cosets", key_faults(), ids=[f[0] for f in key_faults()])
def test_check_pk_matches_the_audit(he_host, orc, name, mutate, max_rows, cosets):
    cs, fixed, copies = key_case()
    E = KeyCheckOracleEngine(he_host, 7, cs.degree())
    pk = plonk.keygen(E, cs, 7, fixed, copies)
    mutate(E, pk)
    got = plonk.check_pk(E, pk, max_rows=max_rows)
    assert got == key_audit(E, pk, plonk.fr_int(orc.srs_tau()), max_rows)
    expected_shape(name, got, pk)


def test_a_key_checked_under_other_params_fails_only_its_commitments(he_host, orc):
    cs, fixed, copies = key_case()
    E = KeyCheckOracleEngine(he_host, 7, cs.degree())
    pk = plonk.keygen(E, cs, 7, fixed, copies)
    other = KeyCheckOracleEngine(he_host, 7, cs.degree(), tau=OTHER_TAU)
    got = plonk.check_pk(other, pk)
    nf, m = cs.num_fixed, len(cs.permutation)
    assert got == [KeyFailure("fixed_commitment", i, None, 1) for i in range(nf)] + [KeyFailure("sigma_commitment", i, None, 1) for i in range(m)]
    assert got == key_audit(other, pk, OTHER_TAU)
    assert plonk.check_pk(other, plonk.keygen(other, cs, 7, fixed, copies)) == []


def test_check_pk_writes_nothing(he_host, orc):
    cs, fixed, copies = key_case()
    E = KeyCheckOracleEngine(he_host, 7, cs.degree())
    pk = plonk.keygen(E, cs, 7, fixed, copies)
    bufs = pk.fixed_values + pk.fixed_polys + pk.fixed_cosets + pk.sigma_values + pk.sigma_polys + pk.sigma_cosets + [pk.l0, pk.l_last, pk.l_active]
    before = [b.a.copy() for b in bufs]
    _bump(E, pk.fixed_values[0], 3)
    before[0] = pk.fixed_values[0].a.copy()
    assert plonk.check_pk(E, pk)
    assert all(np.array_equal(b.a, a) for b, a in zip(bufs, before))


# ---- the checked read -----------------------------------------------------------------------------------------------------
def section_offset(cs, k, ext_k, section, index=0, row=0):
    """byte offset of element `row` of polynomial `index` of a section in write_pk's layout"""
    n, ext, nf, m = 1 << k, 1 << ext_k, cs.num_fixed, len(cs.permutation)
    order = [("l0", 1, ext), ("l_last", 1, ext), ("l_active", 1, ext), ("fixed_values", nf, n), ("fixed_polys", nf, n), ("fixed_cosets", nf, ext),
             ("sigma_values", m, n), ("sigma_polys", m, n), ("sigma_cosets", m, ext)]
    pos = 8 + 64 * (nf + m)
    for name, count, rows in order:
        single = name.startswith("l")
        if not single:
            pos += 4
        if name == section:
            return pos + index * (4 + rows * 32) + 4 + row * 32
        pos += count * (4 + rows * 32)
    raise KeyError(section)


def _patch(path, offset, data):
    with open(path, "r+b") as f:
        f.seek(offset); f.write(data)


PATCHES = [("l0", 0, 5), ("l_last", 0, 0), ("l_active", 0, 511), ("fixed_values", 3, 100), ("fixed_polys", 2, 0), ("fixed_cosets", 1, 257),
           ("sigma_values", 0, 127), ("sigma_polys", 2, 64), ("sigma_cosets", 1, 9)]


def noncanonical_cases():
    """(section, index, row, raw 32 bytes): r, r + 1 and 2^256 - 1 in turn"""
    vals = [R_MOD, R_MOD + 1, (1 << 256) - 1]
    return [(s, i, r, vals[j % 3].to_bytes(32, "little")) for j, (s, i, r) in enumerate(PATCHES)]


def patched_message(path, section, index, row):
    what = section if section.startswith("l") else "%s[%d]" % (section, index)
    return "read_pk: %s: %s row %d: not a canonical field element" % (path, what, row)


def test_checked_read_refuses_a_noncanonical_element_in_every_section(he_host, orc, tmp_path):
    cs, fixed, copies = key_case()
    E = KeyCheckOracleEngine(he_host, 7, cs.degree())
    pk = plonk.keygen(E, cs, 7, fixed, copies)
    clean = str(tmp_path / "clean.pkey")
    plonk.write_pk(E, pk, clean)
    assert plonk.check_pk(E, plonk.read_pk(E, cs, clean, format="RawBytes")) == []
    for section, index, row, raw in noncanonical_cases():
        path = str(tmp_path / ("%s_%d.pkey" % (section, index)))
        with open(clean, "rb") as f, open(path, "wb") as g:
            g.write(f.read())
        _patch(path, section_offset(cs, 7, E.extended_k, section, index, row), raw)
        with pytest.raises(ValueError) as e:
            plonk.read_pk(E, cs, path, format="RawBytes")
        assert str(e.value) == patched_message(path, section, index, row)
        plonk.read_pk(E, cs, path)                                       # the unchecked read believes every byte, as before
        if "cosets" in section or section.startswith("l"):
            plonk.read_pk(E, cs, path, cosets="on_demand", format="RawBytes")   # a lean read never reads the coset sections


def vk_cases(pk):
    """(name, which VK point (index over fixed then sigma), raw 64 bytes, expected reason or None)"""
    def mont(v): return (v * ((1 << 256) % P_MOD) % P_MOD).to_bytes(32, "little")
    x, y = pk.sigma_commitments[1]
    return [("x_is_p", 2, P_MOD.to_bytes(32, "little") + mont(1), "fixed commitment 2: x is not less than the field modulus"),
            ("y_too_big", 0, mont(1) + ((1 << 256) - 1).to_bytes(32, "little"), "fixed commitment 0: y is not less than the field modulus"),
            ("off_curve", pk.cs.num_fixed + 1, mont(x) + mont(y + 1), "sigma commitment 1: not on the curve"),
            ("identity", 1, bytes(64), None)]


def test_checked_read_checks_every_vk_point(he_host, orc, tmp_path):
    cs, fixed, copies = key_case()
    E = KeyCheckOracleEngine(he_host, 7, cs.degree())
    pk = plonk.keygen(E, cs, 7, fixed, copies)
    clean = str(tmp_path / "clean.pkey")
    plonk.write_pk(E, pk, clean)
    for name, which, raw, reason in vk_cases(pk):
        path = str(tmp_path / ("%s.pkey" % name))
        with open(clean, "rb") as f, open(path, "wb") as g:
            g.write(f.read())
        _patch(path, 8 + 64 * which, raw)
        plonk.read_pk(E, cs, path)
        if reason is None:
            got = plonk.read_pk(E, cs, path, format="RawBytes")
            assert got.fixed_commitments[which] == (0, 0)
            assert plonk.check_pk(E, got) == [KeyFailure("fixed_commitment", which, None, 1)]
        else:
            with pytest.raises(ValueError) as e:
                plonk.read_pk(E, cs, path, format="RawBytes")
            assert str(e.value) == "read_pk: %s: %s" % (path, reason)


def test_an_unknown_format_is_refused(he_host, orc, tmp_path):
    cs, fixed, copies = key_case()
    E = KeyCheckOracleEngine(he_host, 7, cs.degree())
    path = str(tmp_path / "k.pkey")
    plonk.write_pk(E, plonk.keygen(E, cs, 7, fixed, copies), path)
    with pytest.raises(ValueError, match="format"):
        plonk.read_pk(E, cs, path, format="Processed")

