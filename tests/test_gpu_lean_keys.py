"""Lean proving keys on the device (keygen / read_pk with cosets="on_demand"): the fixed, sigma and l cosets are rebuilt by the
coset NTT inside create_proof and freed after the quotient. The proofs are byte-identical to a resident key's, the key holds
exactly its n-row data, and no rebuilt coset outlives the proof."""
import json
import os

import pytest

from tests.gpu_common import device_lists

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    """This module's own context, closed when its tests are done. Its K = 23 / K = 24 proofs grow the context's workspaces
    to tens of GiB; a context that lived on for the session would keep them on the device while later test modules, each
    with its own context, prove at K = 24."""
    import torch
    from spectre_b200 import halo2
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    b = halo2.Backend([0])
    yield b
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    b.close()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTANCES = [3, 1, 4, 1, 5]


def _case(shape, k):
    from spectre_b200 import circuits
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, INSTANCES, lookup_bits=4, groups=300)
        return cs, fixed, [adv], copies
    if shape == "wide":
        cs = circuits.wide_shape(3)
        fixed, adv, copies = circuits.wide_witness(cs, k, INSTANCES, lookup_bits=4, groups=300)
        return cs, fixed, adv, copies
    cs = circuits.halo2lib_shape()
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, INSTANCES, lookup_bits=min(16, k - 2), groups=100)
    return cs, fixed, adv, copies


def _allocated(E):
    E.sync()
    return E.torch.cuda.memory_allocated(E.dev)


def _keygen(E, cs, k, fixed, copies, cosets, **kw):
    """-> (key, device bytes the key holds)"""
    from spectre_b200 import plonk
    before = _allocated(E)
    pk = plonk.keygen(E, cs, k, fixed, copies, cosets=cosets, **kw)
    return pk, _allocated(E) - before


def _prove(E, pk, instances, adv, seed):
    """-> proof; asserts that device memory is back at its level before the call"""
    from spectre_b200 import plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    before = _allocated(E)
    proof = plonk.create_proof(E, pk, [instances], adv, SeededRng(seed), EvmTranscriptWrite(pk.vk_digest))
    assert _allocated(E) == before, "create_proof left %d bytes behind" % (_allocated(E) - before)
    return proof


@pytest.mark.parametrize("shape,k", [("aggregation", 12), ("aggregation", 16), ("wide", 13), ("wide", 15), ("halo2lib", 14), ("halo2lib", 16), ("halo2lib", 20)])
def test_lean_key_proves_the_resident_bytes(be, orc, shape, k):
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    cs, fixed, adv, copies = _case(shape, k)
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    lean, lean_bytes = _keygen(E, cs, k, fixed, copies, "on_demand")
    assert lean.lean and lean_bytes == plonk.key_device_bytes(cs, k, E.extended_k, "on_demand")
    proof = _prove(E, lean, INSTANCES, adv, seed=100 + k)
    resident, resident_bytes = _keygen(E, cs, k, fixed, copies, "resident")
    assert resident_bytes == plonk.key_device_bytes(cs, k, E.extended_k, "resident")
    assert (lean.fixed_commitments, lean.sigma_commitments) == (resident.fixed_commitments, resident.sigma_commitments)
    assert _prove(E, resident, INSTANCES, adv, seed=100 + k) == proof
    assert _prove(E, lean, INSTANCES, adv, seed=100 + k) == proof


def test_lean_key_file_on_the_device(be, orc, tmp_path):
    """write_pk of a lean key streams each rebuilt coset through one temporary buffer: the file equals the resident key's;
    read_pk(cosets="on_demand") of it holds only the n-row data and proves the same bytes"""
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    k = 13
    cs, fixed, adv, copies = _case("halo2lib", k)
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    resident, _ = _keygen(E, cs, k, fixed, copies, "resident")
    want = _prove(E, resident, INSTANCES, adv, seed=4)
    paths = [str(tmp_path / name) for name in ("resident.pkey", "lean.pkey")]
    plonk.write_pk(E, resident, paths[0])
    del resident
    lean, _ = _keygen(E, cs, k, fixed, copies, "on_demand")
    before = _allocated(E)
    plonk.write_pk(E, lean, paths[1])
    assert _allocated(E) == before
    with open(paths[0], "rb") as f1, open(paths[1], "rb") as f2:
        assert f1.read() == f2.read()
    del lean
    before = _allocated(E)
    back = plonk.read_pk(E, cs, paths[1], cosets="on_demand")
    assert back.lean and _allocated(E) - before == plonk.key_device_bytes(cs, k, E.extended_k, "on_demand")
    assert _prove(E, back, INSTANCES, adv, seed=4) == want


def _fixture_paths():
    import glob
    return sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "aggregation_k*_proof.json")))


@pytest.mark.parametrize("path", _fixture_paths(), ids=lambda p: p.split("_")[-2])
def test_lean_key_proves_the_contract_accepted_fixture(be, orc, path):
    """K = 23 / K = 24 with a lean key: the bytes of tests/golden/aggregation_k2{3,4}_proof.json, which the reference's
    verifier contracts accepted. The workspaces other tests grew in this context are released first."""
    be.release_workspace()
    import torch
    from spectre_b200 import circuits, plonk
    from spectre_b200.halo2 import ParamsKZG
    with open(path) as f:
        fx = json.load(f)
    k = fx["k"]
    instances = [int(v, 16) for v in fx["instances"]]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, fx["lookup_bits"], fx["groups"], seed=fx["seed"])
    params = ParamsKZG.setup(be, k, orc.srs_tau()).precompute()
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    pk, held = _keygen(E, cs, k, fixed, copies, "on_demand", vk_digest=int(fx["vk_digest"]))
    del fixed
    assert held == plonk.key_device_bytes(cs, k, E.extended_k, "on_demand")
    assert [[hex(x), hex(y)] for x, y in pk.fixed_commitments + pk.sigma_commitments] == fx["vk_points"]
    assert _prove(E, pk, instances, [adv], fx["seed"]).hex() == fx["proof"]
    del E, pk, params
    torch.cuda.empty_cache()


def test_compiled_driver_with_a_lean_key_gives_the_python_bytes(be, orc, tmp_path):
    """tests/cpp/prover_main_lean.cpp (include/spectre_b200_prover.hpp, Cosets::OnDemand, CudaMemory) against
    libspectre_b200.so, proved twice in one process: the Python driver's lean-key bytes"""
    from spectre_b200 import circuits, plonk
    from spectre_b200.halo2 import ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    from tools import cpp_driver
    exe = cpp_driver.build_main_against_the_real_library(str(tmp_path), main="prover_main_lean")
    k, instances = 10, [7, 8, 9]
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=4, groups=40, num_gate_advice=3, num_lookup_advice=2)
    digest = 0x1234567890abcdef1234
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest, cosets="on_demand")
    rec = cpp_driver.RecordingRng(SeededRng(77))
    proof = plonk.create_proof(E, pk, [instances], adv, rec, EvmTranscriptWrite(pk.vk_digest))
    cpp_driver.dump_case(str(tmp_path), "shape halo2lib 3 2", k, digest, instances, copies, rec.counts, fixed, adv, rec.rows, orc.srs_tau())
    rc, log, cproof, _, _ = cpp_driver.run(str(exe), str(tmp_path), repeat=2)
    assert rc == 0, log
    assert cproof == proof


@pytest.mark.parametrize("ids", device_lists())
def test_lean_and_resident_keys_agree_on_several_devices(orc, monkeypatch, ids):
    """one context over several devices: the rebuilt cosets are spread over the devices like every other coset NTT"""
    import torch
    monkeypatch.setenv("SPB_SHARD_MIN_ROWS", "256")
    monkeypatch.setenv("SPB_SHARD_MIN_LOGN", "8")
    from spectre_b200 import circuits, halo2, plonk
    k, instances = 12, [3, 1, 4]
    cs = circuits.halo2lib_shape(4, 1)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=5, groups=200, num_gate_advice=4, num_lookup_advice=1)
    be2 = halo2.Backend(ids)
    try:
        E = plonk.DeviceEngine(be2, halo2.ParamsKZG.setup(be2, k, orc.srs_tau()).precompute(), k, cs.degree())
        proofs = [_prove(E, _keygen(E, cs, k, fixed, copies, cosets)[0], instances, adv, seed=5) for cosets in plonk.COSETS_MODES]
        assert proofs[0] == proofs[1]
    finally:
        torch.cuda.synchronize()
        be2.close()
