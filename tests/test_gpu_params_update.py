"""Powers-of-tau updates on the GPU (ParamsKZG.contribute, plonk.contribute_params, plonk.check_params_updates).

  * exact: setup(k, s) with the trailer of s, then contribute(t), has the points of setup(k, s t), point for point, and the
    trailer ([1]_2, [s t]_2); t = 1 gives the input's points; three updates in a row give setup(k, s t1 t2 t3);
  * a chain of three from the oracle's seed-0 params file at k = 12 passes check_params_updates, its file reads back checked,
    and the final params no longer pass check_params against the seed-0 verifier params;
  * each corrupted chain or final params is reported with its kind and index;
  * on contexts that list device 0 several times, every shard scales its own points and the points are the one-device ones;
  * every error path returns its code, and the input handle is unchanged and still commits correctly;
  * one K = 23 update of the seed-0 params (slow)."""
import ctypes
import random

import numpy as np
import pytest

from spectre_b200 import halo2, plonk
from tests import pypairing as pp
from tests.gpu_common import device_lists
from tests.test_params_check_cpu import doubled, plus_generator, report
from tests.verify_common import contract_vp

pytestmark = pytest.mark.gpu

R = pp.R
GL = halo2.BASIS_G_LAGRANGE
ERR_ARG, ERR_STATE = -2, -4


@pytest.fixture(scope="module")
def be():
    """This module's own context, closed when its tests are done, so the g_to_lagrange workspace of its K = 23 update does not
    stay on the device while later modules prove at K = 24. Handles kept alive by reference cycles are collected first."""
    import gc
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    b = halo2.Backend([0])
    yield b
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    b.close()


def _setup(be, k, s):
    """ParamsKZG::setup under s with the trailer ([1]_2, [s]_2)"""
    params = halo2.ParamsKZG.setup(be, k, plonk.fr_mont(s))
    params.set_g2(pp.g2_limbs(pp.G2_GEN), pp.g2_limbs(pp.g2_mul(pp.G2_GEN, s)))
    return params


def _points(params):
    return params.get_g(), params.get_g(basis=GL)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(_points(a), _points(b)))


def _secrets(seed):
    return [1, 2, R - 1, random.Random(seed).randrange(2, R - 1)]


def _seed0_trailer(orc):
    return pp.g2_limbs(pp.G2_GEN), orc.srs_s_g2().reshape(16)


@pytest.mark.parametrize("k", [0, 1, 2, 5, 10, 16, 20])
def test_an_update_is_setup_under_the_product_of_the_secrets(be, k):
    s = random.Random(k).randrange(2, R)
    params = _setup(be, k, s)
    g2, _ = params.get_g2()
    for t in _secrets(100 + k):
        new = params.contribute(plonk.fr_mont(t))
        assert new.k == k
        assert _same(new, halo2.ParamsKZG.setup(be, k, plonk.fr_mont(s * t % R))), t
        got_g2, got_s_g2 = new.get_g2()
        assert np.array_equal(got_g2, g2) and np.array_equal(got_s_g2, pp.g2_limbs(pp.g2_mul(pp.G2_GEN, s * t % R))), t
        if t == 1:
            assert _same(new, params)
        del new
    if k <= 10:
        ts = [random.Random(200 + i).randrange(2, R) for i in range(3)]
        p = params
        for t in ts:
            p = p.contribute(plonk.fr_mont(t))
        assert _same(p, halo2.ParamsKZG.setup(be, k, plonk.fr_mont(s * ts[0] * ts[1] * ts[2] % R)))


@pytest.fixture(scope="module")
def seed0_chain(be, orc, tmp_path_factory):
    """three contribute_params from the oracle's seed-0 params file at k = 12: (start params, [params after each], records)"""
    path = str(tmp_path_factory.mktemp("params_update") / "kzg_bn254_12.srs")
    orc.write_params_file(path, 12)
    start = halo2.ParamsKZG.read_custom(be, path, "RawBytes")
    chain, updates = [], []
    p = start
    for i in range(3):
        p, u = plonk.contribute_params(be, p)
        chain.append(p)
        updates.append(plonk.ParamsUpdate.from_bytes(u.to_bytes()))
    return start, chain, updates


def _engine(be, params):
    return plonk.DeviceEngine(be, params, params.k, 2)


def test_a_chain_from_the_seed0_params_file_passes(be, orc, kats, seed0_chain, tmp_path):
    start, chain, updates = seed0_chain
    vp = contract_vp(kats)
    assert plonk.check_params(_engine(be, start), be, vp) == []
    final = chain[-1]
    assert plonk.check_params_updates(_engine(be, final), be, vp, updates) == []
    path = str(tmp_path / "contributed.srs")
    final.write(path)
    back = halo2.ParamsKZG.read_custom(be, path, "RawBytes")
    assert _same(back, final) and all(np.array_equal(a, b) for a, b in zip(back.get_g2(), final.get_g2()))
    assert plonk.check_params_updates(_engine(be, back), be, vp, updates) == []
    assert plonk.check_params(_engine(be, back), be) == []
    assert report(plonk.check_params(_engine(be, back), be, vp)) == [("trailer", 1), ("powers", 1)]


def test_each_failure_is_named(be, seed0_chain, kats):
    start, chain, updates = seed0_chain
    vp = contract_vp(kats)
    final = chain[-1]
    u = list(updates)
    g, gl = _points(final)
    g2, s3 = final.get_g2()

    def replaced(g_=g, gl_=gl):
        p = halo2.ParamsKZG.from_parts(be, 12, g_, gl_)
        p.set_g2(g2, s3)
        return p
    other = plonk.prove_params_update(be, u[0].s_g2, u[1].s_g2, 0x5eed, 0x1234)
    end = [("trailer", 1), ("powers", 1)]
    cases = [
        ("t_from_another_t", u[:1] + [u[1]._replace(t_g1=other.t_g1)] + u[2:], final, [("ratio", 1)]),
        ("changed_z", u[:1] + [u[1]._replace(z=(u[1].z + 1) % R)] + u[2:], final, [("knowledge", 1)]),
        ("s_g2_not_t_times_before", u[:2] + [u[2]._replace(s_g2=pp.g2_limbs(pp.g2_add(pp.g2_from_limbs(u[2].s_g2), pp.G2_GEN)))], final,
         [("ratio", 2)] + end),
        ("swapped", [u[0], u[2], u[1]], final, [("ratio", 1), ("ratio", 2)] + end),
        ("identity_t", [u[0]._replace(t_g1=np.zeros(8, np.uint64))] + u[1:], final, [("degenerate", 0)]),
        ("g_replaced", u, replaced(g_=doubled(g, 1000)), [("powers", 1000), ("lagrange", 0)]),
        ("g_lagrange_replaced", u, replaced(gl_=plus_generator(gl, 4095)), [("lagrange", 4095)]),
    ]
    for name, ups, params, want in cases:
        assert report(plonk.check_params_updates(_engine(be, params), be, vp, ups, seed=b"\x11" * 32)) == want, name


@pytest.mark.parametrize("devices", device_lists())
@pytest.mark.parametrize("k", [2, 10])
def test_every_shard_scales_its_own_points(be, devices, k):
    s, t = 0x1234567, 0x89abcdef
    want = _setup(be, k, s).contribute(plonk.fr_mont(t))
    ctx = halo2.Backend(devices)
    try:
        params = _setup(ctx, k, s)
        shards = sum(1 for i in range(len(devices)) if (1 << k) * (i + 1) // len(devices) > (1 << k) * i // len(devices))
        before = ctx.kernel_launches
        got = params.contribute(plonk.fr_mont(t))
        # one scaling launch per non-empty shard, then g_to_lagrange on the first device: lift, powers, k stages, finish
        assert ctx.kernel_launches - before == shards + k + 3
        assert _same(got, want)
        assert all(np.array_equal(a, b) for a, b in zip(got.get_g2(), want.get_g2()))
        del params, got
    finally:
        ctx.close()


def test_error_paths_and_the_input_handle(be, orc):
    lib, c = be.lib, be.ctx
    params = halo2.ParamsKZG.setup(be, 8, orc.srs_tau())
    out = ctypes.c_void_p()
    one = plonk.fr_mont(1)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert lib.spb_srs_contribute(c, params.h, vp(one), ctypes.byref(out)) == ERR_STATE          # no G2 trailer yet
    assert b"trailer" in lib.spb_last_error(c)
    params.set_g2(*_seed0_trailer(orc))
    assert lib.spb_srs_contribute(None, params.h, vp(one), ctypes.byref(out)) == ERR_ARG
    assert lib.spb_srs_contribute(c, None, vp(one), ctypes.byref(out)) == ERR_ARG
    assert lib.spb_srs_contribute(c, params.h, None, ctypes.byref(out)) == ERR_ARG
    assert lib.spb_srs_contribute(c, params.h, vp(one), None) == ERR_ARG
    assert lib.spb_srs_contribute(c, params.h, vp(np.zeros(4, np.uint64)), ctypes.byref(out)) == ERR_ARG
    r_limbs = np.array([(R >> (64 * j)) & ((1 << 64) - 1) for j in range(4)], dtype=np.uint64)
    assert lib.spb_srs_contribute(c, params.h, vp(r_limbs), ctypes.byref(out)) == ERR_ARG
    assert not out.value
    bases = halo2.ParamsKZG.from_bases(be, params.get_g()[:100])
    assert lib.spb_srs_contribute(c, bases.h, vp(one), ctypes.byref(out)) == ERR_STATE
    assert b"plain bases" in lib.spb_last_error(c)
    tables = halo2.ParamsKZG.setup(be, 8, orc.srs_tau())
    tables.set_g2(*_seed0_trailer(orc))
    tables.precompute()
    assert lib.spb_srs_contribute(c, tables.h, vp(one), ctypes.byref(out)) == ERR_STATE
    assert b"spb_srs_precompute" in lib.spb_last_error(c)
    with pytest.raises(halo2.BackendError):
        params.contribute(np.zeros(4, np.uint64))

    before = _points(params) + params.get_g2()
    new, update = plonk.contribute_params(be, params)
    after = _points(params) + params.get_g2()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    poly = orc.fr_random_chacha(1 << 8, 0x0c0)
    assert np.array_equal(orc.g1_to_affine(params.commit(poly)), orc.commit_known_tau(poly))
    assert not np.array_equal(orc.g1_to_affine(new.commit(poly)), orc.g1_to_affine(params.commit(poly)))
    del new
    assert np.array_equal(orc.g1_to_affine(params.commit(poly)), orc.commit_known_tau(poly))


@pytest.mark.slow
def test_a_k23_update_of_the_seed0_params(be, orc):
    tau = plonk.fr_int(orc.srs_tau())
    params = halo2.ParamsKZG.setup(be, 23, orc.srs_tau())
    params.set_g2(*_seed0_trailer(orc))
    t = random.Random(23).randrange(2, R)
    new = params.contribute(plonk.fr_mont(t))
    del params
    assert plonk.check_params(_engine(be, new), be) == []
    assert np.array_equal(new.get_g2()[1], pp.g2_limbs(pp.g2_mul(pp.G2_GEN, tau * t % R)))
    want = halo2.ParamsKZG.setup(be, 23, plonk.fr_mont(tau * t % R))
    n = 1 << 23
    for start in (0, 4321, n // 2 - 7, n - 64):
        for basis in (halo2.BASIS_G, GL):
            assert np.array_equal(new.get_g(start, 64, basis), want.get_g(start, 64, basis)), (start, basis)
