"""The witness check on the device (plonk.check_witness over spb_nonzero_rows_dev, spb_lookup_missing_rows_dev and
spb_copy_mismatches_dev): the reports of the CPU engine and of the pure-Python MockProver (tests/test_witness_check_cpu.py) for
every key mode, exact totals past 2^16 rows, a malformed key named, nothing written, the documented launch counts, and clean
witnesses of Spectre's sizes."""
import numpy as np
import pytest

from tests.test_witness_check_cpu import INSTANCES, WitnessOracleEngine, _build, _case, faults, mock_prover

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    """This module's own context, closed when its tests are done (its K = 23 check grows the lookup workspace)"""
    import torch
    from spectre_b200 import halo2
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    b = halo2.Backend([0])
    yield b
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    b.close()


@pytest.fixture(scope="module")
def he_host(tmp_path_factory):
    return _build(tmp_path_factory, "libhostemu_witness.so", [])


def _engine(be, orc, k, cs):
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    return plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())


def _key(E, cs, k, fixed, copies, mode, tmp_path):
    from spectre_b200 import plonk
    if mode != "read_pk":
        return plonk.keygen(E, cs, k, fixed, copies, cosets=mode)
    path = str(tmp_path / "key.pkey")
    plonk.write_pk(E, plonk.keygen(E, cs, k, fixed, copies), path)
    return plonk.read_pk(E, cs, path)


@pytest.mark.parametrize("mode", ["resident", "on_demand", "per_part", "read_pk"])
def test_device_reports_are_the_cpu_engines(be, orc, he_host, tmp_path, mode):
    from spectre_b200 import plonk
    for name, shape, k, instances, mutate, max_rows in faults():
        cs, fixed, adv, copies = _case(shape, k)
        E = _engine(be, orc, k, cs)
        pk = _key(E, cs, k, fixed, copies, mode, tmp_path)
        assert plonk.check_witness(E, pk, [INSTANCES], adv) == [], name
        adv = [a.copy() for a in adv]
        mutate(adv)
        theta = 0x5eed + k
        got = plonk.check_witness(E, pk, [instances], adv, theta=theta, max_rows=max_rows)
        C = WitnessOracleEngine(he_host, k, cs.degree())
        cpu_key = plonk.keygen(C, cs, k, fixed, copies)
        cpu = plonk.check_witness(C, cpu_key, [instances], adv, theta=theta, max_rows=max_rows)
        assert got == cpu == mock_prover(cpu_key, [instances], adv, max_rows), name
        assert got, name


def test_exact_totals_at_row_zero_past_2_16_and_at_the_last_usable_row(be, orc):
    """k = 18: a column nonzero at three rows, a lookup input missing at them, copies broken at them -- every entry point
    reports exactly those rows, and check_witness names the lookup column's rows"""
    from spectre_b200 import circuits, plonk
    k = 18
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, INSTANCES, lookup_bits=8, groups=50, num_gate_advice=3, num_lookup_advice=2)
    E = _engine(be, orc, k, cs)
    pk = plonk.keygen(E, cs, k, fixed, copies, cosets="on_demand")
    n, u = 1 << k, pk.usable_rows
    rows = [0, (1 << 16) + 77, u - 1]
    col = np.zeros((n, 4), np.uint64)
    for r in rows + [u, n - 1]:                                     # rows >= u are outside the range asked for
        col[r] = plonk.fr_mont(r + 1)
    assert E.nonzero_rows(E.upload(col), 0, u, 16) == (rows, 3)
    assert E.nonzero_rows(E.upload(col), 1, u, 1) == (rows[1:2], 2)
    adv = [a.copy() for a in adv]
    lookup_col = 3                                                  # the first range-lookup column: every usable row a table entry
    for r in rows:
        adv[lookup_col][r] = plonk.fr_mont(1 << 40)
    got = plonk.check_witness(E, pk, [INSTANCES], adv, max_rows=16)
    assert [f for f in got if f.kind == "lookup"] == [plonk.WitnessFailure("lookup", 0, rows, 3)]
    # copies: three cells of column 0 copied to column 1 at the same rows, then column 1 changed there
    vals = [E.upload(np.zeros((n, 4), np.uint64)), E.upload(np.zeros((n, 4), np.uint64))]
    perm = plonk.ConstraintSystem(0, 2, 0, [], [], [("advice", 0), ("advice", 1)])
    sigma = plonk.build_sigma(E, perm, k, [((0, r), (1, r)) for r in rows])
    for r in rows:
        E.write_rows(vals[1], r, plonk.fr_mont(5).reshape(1, 4))
    rep = E.copy_mismatches(vals, sigma, u, 16)
    assert rep == [(3, [(r, 1, r) for r in rows]), (3, [(r, 0, r) for r in rows])]


def test_a_malformed_sigma_entry_is_named(be, orc):
    from spectre_b200 import halo2, plonk
    k = 10
    cs, fixed, adv, copies = _case("wide", k)
    E = _engine(be, orc, k, cs)
    pk = plonk.keygen(E, cs, k, fixed, copies)
    n = 1 << k
    E.write_rows(pk.sigma_values[3], 77, plonk.fr_mont(plonk.DELTA * pow(plonk.omega_of(k), n - 2, plonk.R_MOD)).reshape(1, 4))   # a blinding row
    with pytest.raises(halo2.BackendError, match=r"\(-6\).*column 3, row 77"):
        plonk.check_witness(E, pk, [INSTANCES], adv)
    E.write_rows(pk.sigma_values[1], 5, plonk.fr_mont(12345).reshape(1, 4))                                                     # no label at all
    with pytest.raises(halo2.BackendError, match=r"column 1, row 5"):
        plonk.check_witness(E, pk, [INSTANCES], adv)


def test_a_check_writes_nothing_and_a_later_proof_is_unchanged(be, orc):
    from spectre_b200 import plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    k = 11
    cs, fixed, adv, copies = _case("halo2lib", k)
    E = _engine(be, orc, k, cs)
    pk = plonk.keygen(E, cs, k, fixed, copies)

    def prove():
        return plonk.create_proof(E, pk, [INSTANCES], adv, SeededRng(9), EvmTranscriptWrite(pk.vk_digest))
    want = prove()
    bufs = pk.fixed_values + pk.fixed_polys + pk.fixed_cosets + pk.sigma_values + pk.sigma_polys + pk.sigma_cosets + [pk.l0, pk.l_last, pk.l_active]
    before = [E.download(b).copy() for b in bufs]
    adv_before = [a.copy() for a in adv]
    bad = [a.copy() for a in adv]
    bad[0][9] = plonk.fr_mont(77)
    assert plonk.check_witness(E, pk, [INSTANCES], adv) == []
    assert plonk.check_witness(E, pk, [INSTANCES], bad)
    assert all(np.array_equal(E.download(b), a) for b, a in zip(bufs, before))
    assert all(np.array_equal(a, b) for a, b in zip(adv, adv_before))
    assert prove() == want


def _radix_passes(table_mont, usable):
    """digit passes the lookup sort runs on these values: bytes of each 64-bit limb of the canonical values that not all rows share"""
    from spectre_b200 import plonk
    vals = [plonk.fr_int(r) for r in table_mont[:usable]]
    passes = 0
    for limb in range(4):
        for byte in range(8):
            sh = 64 * limb + 8 * byte
            if len({(v >> sh) & 0xff for v in vals}) > 1:
                passes += 1
    return passes


def test_launch_counts_are_the_documented_ones(be, orc):
    from spectre_b200 import plonk
    k = 12
    n = 1 << k
    E = plonk.DeviceEngine(be, None, k, 4)
    u = n - 7
    rng = np.random.default_rng(5)
    values = E.upload(orc.fr_random_chacha(n, 0x5eed3000))
    L = lambda: be.kernel_launches
    before = L(); E.nonzero_rows(values, 0, u, 16); assert L() - before == 2
    before = L(); assert E.nonzero_rows(values, 9, 9, 16) == ([], 0); assert L() == before
    table = plonk.fr_mont_rows([int(v) for v in rng.integers(0, 1 << 20, size=n)])
    ci, ct = E.upload(plonk.fr_mont_rows([int(v) for v in rng.integers(0, 1 << 21, size=n)])), E.upload(table)
    before = L(); assert E.lookup_missing_rows(ci, ct, u, 16)[1] > 0
    assert L() - before == 12 + 2 * _radix_passes(table, u)
    before = L(); assert E.lookup_missing_rows(ci, ct, 0, 16) == ([], 0); assert L() == before
    perm = plonk.ConstraintSystem(0, 3, 0, [], [], [("advice", c) for c in range(3)])
    sigma = plonk.build_sigma(E, perm, k, [((0, 1), (2, 3))])
    cols = [E.upload(orc.fr_random_chacha(n, 0x5eed3100 + c)) for c in range(3)]
    before = L(); E.copy_mismatches(cols, sigma, u, 4); assert L() - before == 6
    before = L(); assert E.copy_mismatches(cols, sigma, 0, 4) == [(0, []), (0, []), (0, [])]; assert L() == before


@pytest.mark.parametrize("shape,k", [("halo2lib", 20), ("aggregation", 23)])
def test_clean_witnesses_of_spectres_sizes_pass(be, orc, shape, k):
    """the bench's K = 23 aggregation witness (dense) and the k = 20 sync-step witness, on lean keys"""
    be.release_workspace()
    import torch
    from spectre_b200 import circuits, plonk
    inst = list(range(1, 15))
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, min(19, k - 2), 2000, seed=1, dense=True)
        adv = [adv]
    else:
        cs = circuits.halo2lib_shape()
        fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, min(16, k - 2), 500, seed=1)
    E = _engine(be, orc, k, cs)
    pk = plonk.keygen(E, cs, k, fixed, copies, cosets="on_demand")
    del fixed
    assert plonk.check_witness(E, pk, [inst], adv) == []
    del E, pk
    torch.cuda.empty_cache()
