"""spectre_b200.plonk.check_params on the GPU: the device's reports equal the CPU engine's (tests/test_params_check_cpu.py) on the
same corrupted params; seed-0 params pass against the verifier contract's G2 constants with and without window tables, after a
write and a checked read, and after downsize; single bad points at k = 16 are named in either basis, also when they sit in
different shards of a context that lists one device three times; a key made under corrupted params passes check_pk while
check_params names the point; and the check leaves the params, later commitments and torch's allocations as they were."""
import numpy as np
import pytest

from spectre_b200 import circuits, halo2, plonk
from tests import pypairing as pp
from tests.test_params_check_cpu import CheckedPairing, ExplicitEngine, corruption_cases, doubled, plus_generator, report, secret_params, seed0_params
from tests.verify_common import contract_vp

pytestmark = pytest.mark.gpu

GL = halo2.BASIS_G_LAGRANGE


@pytest.fixture(scope="module")
def be():
    """This module's own context, closed when its tests are done: the checks grow the context's MSM, NTT and pairing
    workspaces, which must not stay on the device while later modules prove at K = 24 in the session's context. Handles kept
    alive by reference cycles are collected first, so the context is closed with nothing of theirs left on the device."""
    import gc
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    b = halo2.Backend([0])
    yield b
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    b.close()


def _engine(be, params):
    return plonk.DeviceEngine(be, params, params.k, 2)


def _seed0_trailer(orc):
    return pp.g2_limbs(pp.G2_GEN), orc.srs_s_g2().reshape(16)


def _upload(be, host):
    """a tests.test_params_check_cpu.HostParams as a device handle: from_parts, and set_g2 when it has a trailer"""
    params = halo2.ParamsKZG.from_parts(be, host.k, host.g, host.g_lagrange)
    if host.g2.any():
        params.set_g2(host.g2, host.s_g2)
    return params


def test_device_reports_equal_the_cpu_engines(be, orc, kats):
    vp = contract_vp(kats)
    cases = [(name, host, vp) for name, host, _ in corruption_cases(orc, 4)]
    other = secret_params(orc, 4, 0x1234567)
    cases += [("other_secret_own_trailer", other, None), ("other_secret_contract", other, vp),
              ("other_secret_bare", secret_params(orc, 4, 0x1234567, trailer=False), vp),
              ("s_g2_outside_subgroup", seed0_params(orc, 4), contract_vp(kats, s_g2=pp.g2_twist_point_outside_subgroup()))]
    for i, (name, host, v) in enumerate(cases):
        seed = bytes([i]) * 32
        want = plonk.check_params(ExplicitEngine(host), CheckedPairing(), v, seed=seed)
        got = plonk.check_params(_engine(be, _upload(be, host)), be, v, seed=seed)
        assert got == want, name
    assert report(want) == [("trailer", 1), ("s_g2", 0)]


@pytest.mark.parametrize("k", [16, 20])
def test_seed0_params_pass_with_and_without_tables_and_after_a_checked_read(be, orc, kats, tmp_path, k):
    vp = contract_vp(kats)
    params = halo2.ParamsKZG.setup(be, k, orc.srs_tau())
    E = _engine(be, params)
    assert plonk.check_params(E, be, vp) == []
    params.set_g2(*_seed0_trailer(orc))
    timings = {}
    assert plonk.check_params(E, be, timings=timings) == []
    assert set(timings) == {"points", "powers", "lagrange"}
    path = str(tmp_path / "params.srs")
    params.write(path)
    back = halo2.ParamsKZG.read_custom(be, path, "RawBytes")
    assert plonk.check_params(_engine(be, back), be, vp) == [] and plonk.check_params(_engine(be, back), be) == []
    del back
    params.precompute()
    assert plonk.check_params(E, be, vp) == []


def test_downsized_params_pass(be, orc, kats):
    params = halo2.ParamsKZG.setup(be, 16, orc.srs_tau())
    params.set_g2(*_seed0_trailer(orc))
    small = params.downsize(14)
    assert plonk.check_params(_engine(be, small), be, contract_vp(kats)) == []
    assert plonk.check_params(_engine(be, small), be) == []


@pytest.fixture(scope="module")
def seed0_k16(be, orc):
    params = halo2.ParamsKZG.setup(be, 16, orc.srs_tau())
    return params.get_g(), params.get_g(basis=GL)


@pytest.mark.parametrize("devices,tables", [([0], False), ([0], True), ([0, 0, 0], False)], ids=["one", "tables", "alias3"])
def test_single_bad_points_at_k16_are_named(be, orc, kats, seed0_k16, devices, tables):
    g, gl = seed0_k16
    n = g.shape[0]
    vp = contract_vp(kats)
    ctx = halo2.Backend(devices)
    try:
        for where in (1, n // 2, n - 1):
            for basis in ("g", "g_lagrange"):
                if basis == "g":
                    params = halo2.ParamsKZG.from_parts(ctx, 16, doubled(g, where), gl)
                    want = [("powers", where), ("lagrange", 0)]
                else:
                    params = halo2.ParamsKZG.from_parts(ctx, 16, g, plus_generator(gl, where))
                    want = [("lagrange", where)]
                params.set_g2(*_seed0_trailer(orc))
                if tables:
                    params.precompute()
                assert report(plonk.check_params(_engine(ctx, params), ctx, vp, seed=b"\x5a" * 32)) == want, (basis, where)
                del params
    finally:
        ctx.close()


def test_a_key_under_corrupted_params_passes_check_pk_but_not_check_params(be, orc, kats):
    k, inst = 7, [3, 1, 4]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, lookup_bits=3, groups=20)
    clean = halo2.ParamsKZG.setup(be, k, orc.srs_tau())
    g, gl = clean.get_g(), clean.get_g(basis=GL)
    for bad_g, bad_gl, want in ((g, plus_generator(gl, 5), [("lagrange", 5)]), (doubled(g, 3), gl, [("powers", 3), ("lagrange", 0)])):
        params = halo2.ParamsKZG.from_parts(be, k, bad_g, bad_gl)
        params.set_g2(*_seed0_trailer(orc))
        E = plonk.DeviceEngine(be, params, k, cs.degree())
        pk = plonk.keygen(E, cs, k, fixed, copies)
        assert plonk.check_pk(E, pk) == []
        assert report(plonk.check_params(E, be, contract_vp(kats))) == want


def test_the_check_leaves_params_commitments_and_memory_as_they_were(be, orc, kats, seed0_k16):
    import torch
    g, gl = seed0_k16
    params = halo2.ParamsKZG.from_parts(be, 16, doubled(g, 777), plus_generator(gl, 4321))
    params.set_g2(*_seed0_trailer(orc))
    E = _engine(be, params)
    poly = orc.fr_random_chacha(1 << 16, 0x9a7a)
    before = (params.get_g(), params.get_g(basis=GL), params.commit(poly), params.commit_lagrange(poly))
    torch.cuda.synchronize()
    allocated = torch.cuda.memory_allocated(E.dev)
    assert report(plonk.check_params(E, be, contract_vp(kats))) == [("powers", 777), ("lagrange", 0)]
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(E.dev) == allocated
    after = (params.get_g(), params.get_g(basis=GL), params.commit(poly), params.commit_lagrange(poly))
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    with pytest.raises(ValueError, match="from_bases"):
        plonk.check_params(_engine(be, halo2.ParamsKZG.from_bases(be, g)), be, contract_vp(kats))
