"""Lean proving keys (keygen / read_pk with cosets="on_demand") on the CPU oracle engine: a key that keeps only its n-row data
and rebuilds its extended cosets inside create_proof proves to the same bytes as a resident key, writes the same .pkey file,
and the compiled driver (include/spectre_b200_prover.hpp over the test-only ABI shim) does the same in lean mode."""
import os
import subprocess

import numpy as np
import pytest

from spectre_b200 import circuits, plonk
from spectre_b200.transcript import EvmTranscriptWrite
from tests import plonk_verifier
from tests.plonk_oracle_engine import OracleEngine, SeededRng

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTANCES = [3, 1, 4]


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


def _prove(E, pk, adv, seed=11):
    return plonk.create_proof(E, pk, [INSTANCES], adv, SeededRng(seed), EvmTranscriptWrite(pk.vk_digest))


@pytest.mark.parametrize("shape,k", [("aggregation", 6), ("aggregation", 8), ("wide", 7), ("halo2lib", 8)])
def test_lean_key_proves_the_resident_bytes_and_verifies(orc, shape, k):
    cs, fixed, adv, copies = _case(shape, k)
    E = OracleEngine(k, cs.degree())
    resident = plonk.keygen(E, cs, k, fixed, copies)
    lean = plonk.keygen(E, cs, k, fixed, copies, cosets="on_demand")
    assert not resident.lean and resident.l_polys is None
    assert lean.lean and lean.fixed_cosets is None and lean.sigma_cosets is None and lean.l0 is None and len(lean.l_polys) == 3
    assert (lean.fixed_commitments, lean.sigma_commitments, lean.vk_digest) == (resident.fixed_commitments, resident.sigma_commitments, resident.vk_digest)
    # the coefficient forms a lean key keeps extend to exactly the resident key's cosets
    for p, c in zip(lean.fixed_polys + lean.sigma_polys + lean.l_polys, resident.fixed_cosets + resident.sigma_cosets + [resident.l0, resident.l_last, resident.l_active]):
        assert np.array_equal(E.coeff_to_extended(p).a, c.a)
    proof = _prove(E, lean, adv)
    assert proof == _prove(E, resident, adv)
    assert _prove(E, lean, adv) == proof                         # the key is unchanged by a proof
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    assert plonk_verifier.verify(cs, k, lean.vk_digest, lean.fixed_commitments, lean.sigma_commitments, [INSTANCES], proof, tau)


def test_lean_key_file_is_the_resident_file_and_reads_back_lean(orc, tmp_path):
    k = 7
    cs, fixed, adv, copies = _case("halo2lib", k)
    E = OracleEngine(k, cs.degree())
    resident = plonk.keygen(E, cs, k, fixed, copies)
    lean = plonk.keygen(E, cs, k, fixed, copies, cosets="on_demand")
    paths = [str(tmp_path / name) for name in ("resident.pkey", "lean.pkey")]
    plonk.write_pk(E, resident, paths[0])
    plonk.write_pk(E, lean, paths[1])
    with open(paths[0], "rb") as f1, open(paths[1], "rb") as f2:
        assert f1.read() == f2.read()
    want = _prove(E, resident, adv)
    back = plonk.read_pk(E, cs, paths[1], cosets="on_demand")
    assert back.lean and back.fixed_cosets is None and back.sigma_cosets is None and back.l0 is None
    assert (back.fixed_commitments, back.sigma_commitments, back.vk_digest) == (resident.fixed_commitments, resident.sigma_commitments, resident.vk_digest)
    for a, b in zip(back.fixed_values + back.fixed_polys + back.sigma_values + back.sigma_polys + back.l_polys,
                    lean.fixed_values + lean.fixed_polys + lean.sigma_values + lean.sigma_polys + lean.l_polys):
        assert np.array_equal(a.a, b.a)
    assert _prove(E, back, adv) == want
    assert _prove(E, plonk.read_pk(E, cs, paths[1]), adv) == want    # the same file still reads as a resident key


def test_lean_read_never_reads_the_coset_sections(orc, tmp_path):
    """the engine is asked only for the n-row sections; every coset byte of the file is skipped"""
    k = 6
    cs, fixed, adv, copies = _case("aggregation", k)
    E = OracleEngine(k, cs.degree())
    path = str(tmp_path / "key.pkey")
    plonk.write_pk(E, plonk.keygen(E, cs, k, fixed, copies), path)
    reads = []
    inner = E.read_from_file
    E.read_from_file = lambda p, offset, rows: reads.append(rows) or inner(p, offset, rows)
    plonk.read_pk(E, cs, path, cosets="on_demand")
    assert reads == [1 << k] * (2 * (cs.num_fixed + len(cs.permutation)))


def key_buffers(pk):
    ls = pk.l_polys if pk.lean else [pk.l0, pk.l_last, pk.l_active]
    return pk.fixed_values + pk.fixed_polys + (pk.fixed_cosets or []) + pk.sigma_values + pk.sigma_polys + (pk.sigma_cosets or []) + ls


@pytest.mark.parametrize("cosets", plonk.COSETS_MODES)
def test_key_device_bytes_is_what_a_key_holds(orc, cosets):
    k = 7
    cs, fixed, adv, copies = _case("wide", k)
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, cosets=cosets)
    assert sum(b.a.nbytes for b in key_buffers(pk)) == plonk.key_device_bytes(cs, k, E.extended_k, cosets)


def test_key_device_bytes_at_production_sizes():
    agg, sync = circuits.aggregation_shape(), circuits.halo2lib_shape()
    assert plonk.key_device_bytes(agg, 24, 26) == 27 << 30 and plonk.key_device_bytes(agg, 24, 26, "on_demand") == 17 << 29
    assert plonk.key_device_bytes(agg, 23, 25) == 27 << 29 and plonk.key_device_bytes(agg, 23, 25, "on_demand") == 17 << 28
    assert plonk.key_device_bytes(sync, 20, 22) == 252 << 25 and plonk.key_device_bytes(sync, 20, 22, "on_demand") == 83 << 25


def test_unknown_cosets_mode_is_refused(orc, tmp_path):
    k = 6
    cs, fixed, adv, copies = _case("aggregation", k)
    E = OracleEngine(k, cs.degree())
    with pytest.raises(ValueError, match="cosets"):
        plonk.keygen(E, cs, k, fixed, copies, cosets="lean")
    with pytest.raises(ValueError, match="cosets"):
        plonk.read_pk(E, cs, str(tmp_path / "none.pkey"), cosets=None)


# ---- the compiled driver in lean mode over the CPU shim of the C ABI -----------------------------------------------------
def build_lean_main_over_the_shim(out_dir):
    """tests/cpp/prover_main_lean.cpp linked against tests/abi_shim (the oracle behind the C ABI), built into out_dir"""
    from oracle import oracle as orc
    orc.build()
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    shim = os.path.join(out_dir, "libspb_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", shim, os.path.join(ROOT, "tests", "abi_shim", "shim.cpp"),
                           "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    exe = os.path.join(out_dir, "prover_main_lean")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "prover_main_lean.cpp"), "-L" + out_dir, "-lspb_shim",
                           "-Wl,-rpath," + out_dir, "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    return exe


@pytest.mark.parametrize("shape,k", [("aggregation", 7), ("halo2lib", 8)])
def test_cpp_driver_with_a_lean_key_reproduces_the_python_proof(orc, tmp_path, shape, k):
    from tools import cpp_driver
    exe = build_lean_main_over_the_shim(str(tmp_path))
    cs, fixed, adv, copies = _case(shape, k)
    digest = 0x1234567890abcdef1234
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest, cosets="on_demand")
    rec = cpp_driver.RecordingRng(SeededRng(77))
    proof = plonk.create_proof(E, pk, [INSTANCES], adv, rec, EvmTranscriptWrite(pk.vk_digest))
    case = tmp_path / "case"
    case.mkdir()
    head = "shape aggregation" if shape == "aggregation" else "shape halo2lib 3 2"
    cpp_driver.dump_case(str(case), head, k, digest, INSTANCES, copies, rec.counts, fixed, adv, rec.rows, orc.srs_tau())
    rc, log, cproof, _, _ = cpp_driver.run(exe, str(case), repeat=2)
    assert rc == 0, log
    assert cproof == proof
