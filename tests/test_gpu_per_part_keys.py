"""Per-part proving keys on the device (cosets="per_part"): create_proof builds every coset one n-row part at a time with
spb_coeff_to_extended_part_batch_dev, evaluates the quotient terms on the part and scatters it into the extended `values`.
The part kernels equal the whole-coset kernels sliced [j::R] bit for bit, the proofs are byte-identical to a resident key's
and to the contract-accepted fixtures, and no buffer but `values` and the quotient's coefficients exceeds n rows."""
import json
import os

import numpy as np
import pytest

from tests.gpu_common import device_lists

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTANCES = [3, 1, 4, 1, 5]


@pytest.fixture(scope="module")
def be():
    """This module's own context, closed when its tests are done: its K = 23 / K = 24 proofs grow the context's workspaces, which
    must not stay on the device while later modules prove in their own contexts."""
    import torch
    from spectre_b200 import halo2
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    b = halo2.Backend([0])
    yield b
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    b.close()


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


def _prove(E, pk, instances, adv, seed):
    """-> proof; asserts that device memory is back at its level before the call"""
    from spectre_b200 import plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    before = _allocated(E)
    proof = plonk.create_proof(E, pk, [instances], adv, SeededRng(seed), EvmTranscriptWrite(pk.vk_digest))
    assert _allocated(E) == before, "create_proof left %d bytes behind" % (_allocated(E) - before)
    return proof


def _engine(be, k, j):
    from spectre_b200 import plonk
    return plonk.DeviceEngine(be, None, k, j)


def _g(part, extended_k):
    from spectre_b200 import plonk
    return plonk.fr_mont(plonk.ZETA * pow(plonk.omega_of(extended_k), part, plonk.R_MOD))


# ---- kernels ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("j,k,count", [(3, 6, 3), (5, 10, 2), (9, 11, 3), (3, 14, 2), (5, 17, 2), (9, 20, 2)])
def test_part_transform_is_the_whole_coset_sliced(be, orc, j, k, count):
    """R = 2, 4, 8; one-pass plans (k <= 11, two-level twiddles below k = 12) up to 2^20; every part of every polynomial of a batch"""
    E = _engine(be, k, j)
    n, R = 1 << k, 1 << (E.extended_k - k)
    assert R == {3: 2, 5: 4, 9: 8}[j]
    coeffs = [orc.fr_random_chacha(n, 0x5eed1000 + 16 * k + i) for i in range(count)]
    polys = [E.upload(c) for c in coeffs]
    whole = [E.download(E.coeff_to_extended(p)) for p in polys]
    outs = [E.alloc_uninit(n) for _ in polys]
    for part in range(R):
        E.coeff_to_extended_part_many(polys, part, outs)
        for i in range(count):
            assert np.array_equal(E.download(outs[i]), whole[i][part::R]), "part %d of %d, polynomial %d, k = %d" % (part, R, i, k)
    for p, c in zip(polys, coeffs):
        assert np.array_equal(E.download(p), c)                      # out of place: the coefficients are untouched


def test_part_scatter_is_exact_and_refuses_a_part_past_r(be, orc):
    from spectre_b200 import halo2
    k = 12
    E = _engine(be, k, 5)
    n, R = 1 << k, 1 << (E.extended_k - k)
    parts = [orc.fr_random_chacha(n, 0x5eed1100 + j) for j in range(R)]
    values = E.alloc(R * n)
    for j, p in enumerate(parts):
        E.extended_part_scatter(E.upload(p), j, values)
    got = E.download(values)
    for j, p in enumerate(parts):
        assert np.array_equal(got[j::R], p)
    with pytest.raises(halo2.BackendError):
        E.extended_part_scatter(E.upload(parts[0]), R, values)
    with pytest.raises(halo2.BackendError):
        E.coeff_to_extended_part_many([E.upload(parts[0])], R, [E.alloc(n)])


def test_quotient_passes_on_parts_are_the_whole_coset_passes_sliced(be, orc):
    """spb_graph_evaluate_dev, the coset permutation entry point and spb_lookup_constraints_dev on sliced inputs (size n, rot_scale 1,
    g_j) equal the whole-coset passes sliced [j::R]; the coset entry point with (zeta, extended_omega) is spb_permutation_constraints_dev"""
    from spectre_b200 import circuits, plonk
    k = 11
    cs = circuits.halo2lib_shape(3, 2)
    E = _engine(be, k, cs.degree())
    n, ek = 1 << k, E.extended_k
    R, ext = 1 << (ek - k), 1 << ek
    seed = [0x5eed1200]

    def rnd(rows):
        seed[0] += 1
        return orc.fr_random_chacha(rows, seed[0])
    fixed, advice, inst = [rnd(ext) for _ in range(cs.num_fixed)], [rnd(ext) for _ in range(cs.num_advice)], [rnd(ext) for _ in range(cs.num_instance)]
    z, cols, sigma = [rnd(ext) for _ in range(2)], [rnd(ext) for _ in range(5)], [rnd(ext) for _ in range(5)]
    l0, l_last, l_active, start = rnd(ext), rnd(ext), rnd(ext), rnd(ext)
    product, pin, ptab = rnd(ext), rnd(ext), rnd(ext)
    beta, gamma, theta, y = (rnd(1)[0] for _ in range(4))
    ext_omega = plonk.fr_mont(plonk.omega_of(ek))
    up = lambda arrs: [E.upload(a) for a in arrs]

    def passes(sl, size, rot_scale, g, omega):
        """gates, then the permutation, then one lookup, on the rows `sl` of every input"""
        F, A, I = up([a[sl] for a in fixed]), up([a[sl] for a in advice]), up([a[sl] for a in inst])
        Z, C, S = up([a[sl] for a in z]), up([a[sl] for a in cols]), up([a[sl] for a in sigma])
        L0, LL, LA, P, PI, PT = up([a[sl] for a in (l0, l_last, l_active, product, pin, ptab)])
        values, table_value = E.upload(start[sl]), E.alloc(size)
        E.graph_evaluate(cs.gates_program(), F, A, I, beta, gamma, theta, y, values, size, rot_scale)
        E.permutation_constraints(values, size, rot_scale, -4, 2, Z, C, S, L0, LL, LA, beta, gamma, y, omega, coset_generator=g)
        E.graph_evaluate(cs.lookup_value_program(0), F, A, I, beta, gamma, theta, plonk.fr_mont(0), table_value, size, rot_scale)
        E.lookup_constraints(values, size, rot_scale, P, PI, PT, table_value, L0, LL, LA, beta, gamma, y)
        return E.download(values)
    whole = passes(slice(None), ext, R, None, ext_omega)
    assert np.array_equal(passes(slice(None), ext, R, plonk.fr_mont(plonk.ZETA), ext_omega), whole)
    omega = plonk.fr_mont(plonk.omega_of(k))
    for j in range(R):
        assert np.array_equal(passes(slice(j, None, R), n, 1, _g(j, ek), omega), whole[j::R]), "part %d of %d" % (j, R)


# ---- proofs ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,k", [("aggregation", 12), ("aggregation", 16), ("wide", 13), ("wide", 15), ("halo2lib", 14), ("halo2lib", 16), ("halo2lib", 20)])
def test_per_part_key_proves_the_resident_bytes(be, orc, shape, k):
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    cs, fixed, adv, copies = _case(shape, k)
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    before = _allocated(E)
    per_part = plonk.keygen(E, cs, k, fixed, copies, cosets="per_part")
    assert per_part.lean and per_part.per_part
    assert _allocated(E) - before == plonk.key_device_bytes(cs, k, E.extended_k, "per_part")
    proof = _prove(E, per_part, INSTANCES, adv, seed=100 + k)
    resident = plonk.keygen(E, cs, k, fixed, copies)
    assert _prove(E, resident, INSTANCES, adv, seed=100 + k) == proof
    assert _prove(E, per_part, INSTANCES, adv, seed=100 + k) == proof


def test_per_part_proof_holds_no_extended_buffer_but_values_and_h(be, orc):
    """every engine allocation of a per-part create_proof has at most n rows, except the one extended `values` and the quotient's
    n (d - 1) coefficients; memory returns to its level, and the peak is below an on_demand proof's"""
    import torch
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    k = 16
    cs, fixed, adv, copies = _case("aggregation", k)
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    n, ext = 1 << k, 1 << E.extended_k
    keys = {mode: plonk.keygen(E, cs, k, fixed, copies, cosets=mode) for mode in ("on_demand", "per_part")}
    _prove(E, keys["per_part"], INSTANCES, adv, seed=3)             # warm: the library's workspaces reach their size
    rows = []
    inner = {name: getattr(E, name) for name in ("alloc", "alloc_uninit")}
    for name, fn in inner.items():
        setattr(E, name, lambda r, fn=fn: rows.append(r) or fn(r))
    try:
        peaks = {}
        for mode in ("per_part", "on_demand"):
            rows.clear()
            E.sync(); torch.cuda.reset_peak_memory_stats(E.dev)
            base = torch.cuda.memory_allocated(E.dev)
            _prove(E, keys[mode], INSTANCES, adv, seed=3)
            peaks[mode] = torch.cuda.max_memory_allocated(E.dev) - base
            if mode == "per_part":
                large = sorted(r for r in rows if r > n)
                assert large == sorted([ext, n * (cs.degree() - 1)]), large
    finally:
        for name, fn in inner.items():
            setattr(E, name, fn)
    assert peaks["per_part"] < peaks["on_demand"], peaks


def _fixture_paths():
    import glob
    return sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "aggregation_k*_proof.json")))


@pytest.mark.parametrize("path", _fixture_paths(), ids=lambda p: p.split("_")[-2])
def test_per_part_key_proves_the_contract_accepted_fixture(be, orc, path):
    """K = 23 / K = 24 with a per-part key: the bytes of tests/golden/aggregation_k2{3,4}_proof.json, which the reference's
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
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=int(fx["vk_digest"]), cosets="per_part")
    del fixed
    assert [[hex(x), hex(y)] for x, y in pk.fixed_commitments + pk.sigma_commitments] == fx["vk_points"]
    assert _prove(E, pk, instances, [adv], fx["seed"]).hex() == fx["proof"]
    del E, pk, params
    torch.cuda.empty_cache()


def test_compiled_driver_with_a_per_part_key_gives_the_python_bytes(be, orc, tmp_path):
    """tests/cpp/prover_main_per_part.cpp (include/spectre_b200_prover.hpp, Cosets::PerPart, CudaMemory) against
    libspectre_b200.so, proved twice in one process: the Python driver's per-part bytes"""
    from spectre_b200 import circuits, plonk
    from spectre_b200.halo2 import ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    from tools import cpp_driver
    exe = cpp_driver.build_main_against_the_real_library(str(tmp_path), main="prover_main_per_part")
    k, instances = 10, [7, 8, 9]
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=4, groups=40, num_gate_advice=3, num_lookup_advice=2)
    digest = 0x1234567890abcdef1234
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest, cosets="per_part")
    rec = cpp_driver.RecordingRng(SeededRng(77))
    proof = plonk.create_proof(E, pk, [instances], adv, rec, EvmTranscriptWrite(pk.vk_digest))
    cpp_driver.dump_case(str(tmp_path), "shape halo2lib 3 2", k, digest, instances, copies, rec.counts, fixed, adv, rec.rows, orc.srs_tau())
    rc, log, cproof, _, _ = cpp_driver.run(str(exe), str(tmp_path), repeat=2)
    assert rc == 0, log
    assert cproof == proof


@pytest.mark.parametrize("ids", device_lists())
def test_per_part_and_resident_keys_agree_on_several_devices(orc, monkeypatch, ids):
    """one context over several devices: the part transforms are spread over the devices and the part passes and scatter are
    sharded by rows"""
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
        proofs = [_prove(E, plonk.keygen(E, cs, k, fixed, copies, cosets=mode), instances, adv, seed=5) for mode in ("resident", "per_part")]
        assert proofs[0] == proofs[1]
    finally:
        torch.cuda.synchronize()
        be2.close()
