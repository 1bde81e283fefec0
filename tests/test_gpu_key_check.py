"""The proving-key check on the device (plonk.check_pk over spb_sigma_check_dev, the checked plonk.read_pk over
spb_fr_first_noncanonical_dev): the reports of the CPU engine and of the pure-Python audit (tests/test_key_check_cpu.py) for every
key mode, a key checked under other params, the same error texts from the checked read, exact totals past 2^16 rows, nothing
written, the documented launch counts, and clean keys of Spectre's sizes."""
import numpy as np
import pytest

from tests.test_key_check_cpu import (OTHER_TAU, KeyCheckOracleEngine, _build, _label, _patch, he_sigma_check, key_audit, key_case, key_faults,
                                      noncanonical_cases, patched_message, section_offset, vk_cases)

pytestmark = pytest.mark.gpu
K = 7


@pytest.fixture(scope="module")
def be():
    """This module's own context, closed when its tests are done (its K = 23 key grows the context's workspaces)"""
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
    return _build(tmp_path_factory, "libhostemu_key_check.so", [])


def _engine(be, orc, k, cs, tau=None):
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    return plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau() if tau is None else plonk.fr_mont(tau)), k, cs.degree())


def _key(E, cs, k, fixed, copies, mode, tmp_path):
    from spectre_b200 import plonk
    if mode != "read_pk":
        return plonk.keygen(E, cs, k, fixed, copies, cosets=mode)
    path = str(tmp_path / "key.pkey")
    plonk.write_pk(E, plonk.keygen(E, cs, k, fixed, copies), path)
    return plonk.read_pk(E, cs, path, format="RawBytes")


@pytest.mark.parametrize("mode", ["resident", "on_demand", "per_part", "read_pk"])
def test_device_reports_are_the_cpu_engines(be, orc, he_host, tmp_path, mode):
    from spectre_b200 import plonk
    cs, fixed, copies = key_case(K)
    E = _engine(be, orc, K, cs)
    for name, mutate, max_rows, cosets in key_faults():
        pk = _key(E, cs, K, fixed, copies, mode, tmp_path)
        if cosets and pk.lean:
            continue
        mutate(E, pk)
        got = plonk.check_pk(E, pk, max_rows=max_rows)
        C = KeyCheckOracleEngine(he_host, K, cs.degree())
        cpu_key = plonk.keygen(C, cs, K, fixed, copies, cosets="resident" if mode == "read_pk" else mode)
        mutate(C, cpu_key)
        cpu = plonk.check_pk(C, cpu_key, max_rows=max_rows)
        assert got == cpu, name
        if not pk.lean:
            assert got == key_audit(C, cpu_key, plonk.fr_int(orc.srs_tau()), max_rows), name
        assert (got == []) == (name == "clean"), name


def test_a_key_checked_under_other_params_fails_exactly_its_commitments(be, orc, he_host):
    from spectre_b200 import plonk
    from spectre_b200.plonk import KeyFailure
    cs, fixed, copies = key_case(K)
    pk = plonk.keygen(_engine(be, orc, K, cs), cs, K, fixed, copies)
    other = _engine(be, orc, K, cs, tau=OTHER_TAU)
    got = plonk.check_pk(other, pk)
    nf, m = cs.num_fixed, len(cs.permutation)
    assert got == [KeyFailure("fixed_commitment", i, None, 1) for i in range(nf)] + [KeyFailure("sigma_commitment", i, None, 1) for i in range(m)]
    C = KeyCheckOracleEngine(he_host, K, cs.degree(), tau=OTHER_TAU)
    assert got == plonk.check_pk(C, plonk.keygen(KeyCheckOracleEngine(he_host, K, cs.degree()), cs, K, fixed, copies))
    assert plonk.check_pk(other, plonk.keygen(other, cs, K, fixed, copies)) == []


def test_the_checked_read_gives_the_cpu_engines_error_texts(be, orc, he_host, tmp_path):
    from spectre_b200 import plonk
    cs, fixed, copies = key_case(K)
    E = _engine(be, orc, K, cs)
    C = KeyCheckOracleEngine(he_host, K, cs.degree())
    pk = plonk.keygen(E, cs, K, fixed, copies)
    clean = str(tmp_path / "clean.pkey")
    plonk.write_pk(E, pk, clean)
    cases = [(str(tmp_path / ("%s_%d.pkey" % (s, i))), section_offset(cs, K, E.extended_k, s, i, r), raw, patched_message(str(tmp_path / ("%s_%d.pkey" % (s, i))), s, i, r))
             for s, i, r, raw in noncanonical_cases()]
    cases += [(str(tmp_path / ("%s.pkey" % name)), 8 + 64 * which, raw, None if reason is None else "read_pk: %s: %s" % (str(tmp_path / ("%s.pkey" % name)), reason))
              for name, which, raw, reason in vk_cases(pk)]
    for path, offset, raw, message in cases:
        with open(clean, "rb") as f, open(path, "wb") as g:
            g.write(f.read())
        _patch(path, offset, raw)
        for engine in (E, C):
            if message is None:
                plonk.read_pk(engine, cs, path, format="RawBytes")
                continue
            with pytest.raises(ValueError) as e:
                plonk.read_pk(engine, cs, path, format="RawBytes")
            assert str(e.value) == message
        plonk.read_pk(E, cs, path)
    assert plonk.check_pk(E, plonk.read_pk(E, cs, clean, format="RawBytes")) == []


def test_sigma_check_exact_totals_at_row_zero_past_2_16_and_at_the_last_usable_row(be, orc, he_host):
    """k = 18: failures of every kind at row 0, past 2^16 and at u - 1, reported exactly and identically twice"""
    from spectre_b200 import plonk
    k, cols = 18, 3
    n = 1 << k
    u = n - 7
    E = plonk.DeviceEngine(be, None, k, 4)
    perm = plonk.ConstraintSystem(0, cols, 0, [], [], [("advice", c) for c in range(cols)])
    rows = [0, (1 << 16) + 77, u - 1]
    sigma = plonk.build_sigma(E, perm, k, [((0, r), (2, r + 1)) for r in range(1, 1 << 17, 97)])
    for r in rows:
        E.write_rows(sigma[0], r, plonk.fr_mont(r * 7919 + 5).reshape(1, 4))      # labels nothing: kind 0, and its cell unlabelled
        E.write_rows(sigma[1], r, _label(k, 2, n - 2))                             # labels a blinding row: kind 0
    E.write_rows(sigma[2], u + 1, _label(k, 0, 9))                                 # a blinding row moved: kind 1
    first = E.sigma_check(sigma, u, 16)
    assert E.sigma_check(sigma, u, 16) == first
    assert first == he_sigma_check(he_host, k, [E.download(s) for s in sigma], u, 16)
    assert first[0][0] == (3, rows) and first[1][0] == (3, rows) and first[2][1] == (1, [u + 1])
    assert first[0][2] == (3, rows) and first[1][2] == (3, rows) and first[2][2] == (1, [u + 1])
    assert first[0][1] == first[1][1] == (0, []) and first[2][0] == (0, [])
    assert E.sigma_check(sigma, u, 2)[0][0] == (3, rows[:2])


def test_launch_counts_are_the_documented_ones(be, orc):
    from spectre_b200 import plonk
    k = 12
    n = 1 << k
    E = plonk.DeviceEngine(be, None, k, 4)
    L = lambda: be.kernel_launches
    values = E.upload(orc.fr_random_chacha(n, 0x5eed4000))
    before = L(); assert E.first_noncanonical(values, n) == n; assert L() - before == 1
    before = L(); assert E.first_noncanonical(values, 0) == 0; assert L() == before
    perm = plonk.ConstraintSystem(0, 3, 0, [], [], [("advice", c) for c in range(3)])
    sigma = plonk.build_sigma(E, perm, k, [((0, 1), (2, 3))])
    before = L(); assert E.sigma_check(sigma, n - 7, 4) == [[(0, [])] * 3] * 3; assert L() - before == 7 * 3
    before = L(); E.sigma_check(sigma, n, 4); assert L() - before == 5 * 3
    before = L(); E.sigma_check(sigma, 0, 4); assert L() - before == 5 * 3
    before = L(); assert be.sigma_check_dev(k, [], n - 7, 4) == []; assert L() == before


def test_a_check_writes_nothing_and_a_later_proof_is_unchanged(be, orc):
    from spectre_b200 import plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    from tests.test_witness_check_cpu import INSTANCES, _case
    k = 11
    cs, fixed, adv, copies = _case("halo2lib", k)
    E = _engine(be, orc, k, cs)
    pk = plonk.keygen(E, cs, k, fixed, copies)

    def prove():
        return plonk.create_proof(E, pk, [INSTANCES], adv, SeededRng(9), EvmTranscriptWrite(pk.vk_digest))
    want = prove()
    bufs = pk.fixed_values + pk.fixed_polys + pk.fixed_cosets + pk.sigma_values + pk.sigma_polys + pk.sigma_cosets + [pk.l0, pk.l_last, pk.l_active]
    before = [E.download(b).copy() for b in bufs]
    assert plonk.check_pk(E, pk) == []
    assert all(np.array_equal(E.download(b), a) for b, a in zip(bufs, before))
    assert prove() == want


@pytest.mark.parametrize("shape,k", [("halo2lib", 20), ("aggregation", 23)])
def test_clean_keys_of_spectres_sizes_pass(be, orc, tmp_path, shape, k):
    """the k = 20 sync-step key and the K = 23 aggregation key: check_pk on the resident key, then the checked read of its file
    and check_pk on what it read"""
    be.release_workspace()
    import torch
    from spectre_b200 import circuits, plonk
    inst = list(range(1, 15))
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, _, copies = circuits.aggregation_witness(cs, k, inst, min(19, k - 2), 2000, seed=1, dense=True)
    else:
        cs = circuits.halo2lib_shape()
        fixed, _, copies = circuits.halo2lib_witness(cs, k, inst, min(16, k - 2), 500, seed=1)
    E = _engine(be, orc, k, cs)
    pk = plonk.keygen(E, cs, k, fixed, copies)
    del fixed
    assert plonk.check_pk(E, pk) == []
    path = str(tmp_path / "key.pkey")
    plonk.write_pk(E, pk, path)
    del pk
    torch.cuda.empty_cache()
    assert plonk.check_pk(E, plonk.read_pk(E, cs, path, format="RawBytes")) == []
    del E
    be.release_workspace()
    torch.cuda.empty_cache()
