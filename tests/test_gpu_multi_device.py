"""The multi-device paths on one GPU: contexts that list device 0 two, three, four, eight (and 32) times.

Each entry of such a context has its own stream, events, workspaces, MSM lanes, twiddle tables and SRS shard, and its work
runs concurrently with the other entries', as it would on separate GPUs; every host loop, index calculation, seed chain, event
dependency and peer copy of the multi-device code runs for real. Every comparison is bit-exact: with the CPU oracle, with the
known-secret commitment of the seed-0 SRS, or with the same call on a one-device context. The sharding thresholds are lowered
through SPB_SHARD_MIN_ROWS / SPB_SHARD_MIN_LOGN so that small inputs take the sharded paths, and `spb_kernel_launches` deltas
show that they did: a context that silently fell back to one device would compute the same values.

What aliasing cannot show -- a launch or allocation on the wrong physical device, a missing cudaSetDevice, missing peer
enablement, NVLink speed -- needs two real GPUs, where tests/test_gpu_{ntt,msm,plonk,...}.py run their multi-device tests
on the real devices too (tests/gpu_common.py::device_lists).

`pytest -s` prints the device memory in use after the G = 8 cases (the library's workspaces and tables are grow-only caches,
so that is their peak)."""
import functools

import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be  # noqa: F401
from tests.test_gpu_scale import _graph_case, _npass, _residues

pytestmark = pytest.mark.gpu

R = pyref.R_MOD
GS = [2, 3, 8]
_contexts = {}
_mem_used = {}


def _ctx(G):
    """the module's context over device 0 listed G times"""
    if G not in _contexts:
        from spectre_b200 import halo2
        _contexts[G] = halo2.Backend([0] * G)
    return _contexts[G]


@pytest.fixture(scope="module", autouse=True)
def _close_contexts(be):
    """every aliased context multiplies the per-device caches on one card: free them so that later modules' K = 24 proofs fit"""
    yield
    import torch
    for cache in (_ntt_case, _one_device_params, _aliased_params, _columns, _one_device_proof):
        cache.cache_clear()
    for b in _contexts.values():
        b.release_workspace()
        b.close()
    _contexts.clear()
    be.release_workspace()
    torch.cuda.empty_cache()
    for G, used in sorted(_mem_used.items()):
        print("aliased contexts: %.2f GiB of device memory in use after the G = %d cases" % (used / 2 ** 30, G))


@pytest.fixture(autouse=True)
def _record_memory(request):
    yield
    G = getattr(request.node, "callspec", None) and request.node.callspec.params.get("G")
    if G == 8:
        import torch
        free, total = torch.cuda.mem_get_info(0)
        _mem_used[G] = max(_mem_used.get(G, 0), total - free)


@pytest.fixture
def shard_small(monkeypatch):
    """the lowest thresholds: row passes shard from 256 rows, batch NTTs from 2^8 points"""
    monkeypatch.setenv("SPB_SHARD_MIN_ROWS", "256")
    monkeypatch.setenv("SPB_SHARD_MIN_LOGN", "8")


def _up(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def _down(t):
    return t.cpu().numpy().view(np.uint64)


def _counted(b, call):
    before = b.kernel_launches
    out = call()
    return b.kernel_launches - before, out


def _row_ranges(G, rows):
    """csrc/capi.cu row_ranges at SPB_SHARD_MIN_ROWS = 256: (lo, hi) of the non-empty ranges of G devices"""
    if G < 2 or rows < 256:
        return [(0, rows)]
    per = ((rows + G - 1) // G + 255) // 256 * 256
    return [(per * i, min(per * (i + 1), rows)) for i in range(G) if per * i < rows]


def _fraction_product_launches(G, rows):
    """plonk.cu fraction_product: one range runs the terms kernel, three batch-inversion kernels, the product pass and three
    scan kernels (8); with several ranges each also runs the two total-product kernels of its range total (10 per range)"""
    n_ranges = len(_row_ranges(G, rows))
    return 8 if n_ranges == 1 else 10 * n_ranges


# ---- the context itself ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", GS)
def test_aliased_context_starts_without_an_error(orc, G):
    """spb_init on an aliased list leaves no error behind: its first call (a checked launch) succeeds, and spb_last_error stays
    empty"""
    from spectre_b200 import halo2
    b = halo2.Backend([0] * G)
    try:
        assert b.lib.spb_last_error(b.ctx) == b""
        a, c = orc.fr_random_chacha(1000, 1), orc.fr_random_chacha(1000, 2)
        assert np.array_equal(b.vec_mul(a, c), orc.fr([x * y % R for x, y in zip(orc.fr_ints(a), orc.fr_ints(c))]))
        assert b.lib.spb_last_error(b.ctx) == b""
    finally:
        b.close()


# ---- row-range grand products ------------------------------------------------------------------------------------------
LOOKUP_ROWS = [256, 257, "256G+1", (1 << 16) + 3]


@pytest.mark.parametrize("rows", LOOKUP_ROWS, ids=str)
@pytest.mark.parametrize("G", GS)
def test_lookup_product_by_row_range(orc, shard_small, G, rows):
    """spb_lookup_product_dev per row range, range totals chained into the seeds; a zero denominator (permuted table + gamma = 0)
    sits in the second range where there is one. At 256 rows there is one range; at 257 rows on 8 devices every range after the
    second is empty."""
    b = _ctx(G)
    n = 256 * G + 1 if rows == "256G+1" else rows
    ranges = _row_ranges(G, n)
    n_blinds = 5
    arrs = [orc.fr_random_chacha(n, 0x700 + 4 * n + i) for i in range(4)]
    beta, gamma = orc.fr_random_chacha(2, 0x7ff + n)
    zero_row = ranges[1][0] + 1 if len(ranges) > 1 and ranges[1][0] + 1 < n - n_blinds - 1 else 9
    arrs[3][zero_row] = orc.fr([-orc.fr_ints(gamma.reshape(1, 4))[0]])[0]
    blinds = orc.fr_random_chacha(n_blinds, 0x7fe).reshape(-1, 4)
    d = [_up(a) for a in arrs]
    dz = _up(np.zeros((n, 4), np.uint64))
    launches, _ = _counted(b, lambda: b.lookup_product_dev(n, *[t.data_ptr() for t in d], beta, gamma, blinds, dz.data_ptr()))
    assert np.array_equal(_down(dz), orc.lookup_product(*arrs, beta, gamma, blinds))
    assert launches == _fraction_product_launches(G, n), (launches, ranges)


@pytest.mark.parametrize("k,n_blinds", [(8, 5), (9, 0), (16, 5)])
@pytest.mark.parametrize("G", GS)
def test_permutation_product_by_row_range(orc, shard_small, G, k, n_blinds):
    """spb_permutation_product_dev over three sets of a 5-column permutation, last_z chained from set to set; with no blinding
    rows the last row of z is the chained value, so a range that stops short shows"""
    b = _ctx(G)
    n, n_cols, chunk = 1 << k, 5, 2
    values = [orc.fr_random_chacha(n, 0x800 + c) for c in range(n_cols)]
    sigma = [orc.fr_random_chacha(n, 0x900 + c) for c in range(n_cols)]
    values[0][3] = 0; sigma[0][5] = 0
    beta, gamma = orc.fr_random_chacha(2, 0xa00 + k)
    dv, ds = [_up(a) for a in values], [_up(a) for a in sigma]
    dz = _up(np.zeros((n, 4), np.uint64))
    last_o = last_g = orc.fr([1])[0]
    for s, lo in enumerate(range(0, n_cols, chunk)):
        hi = min(lo + chunk, n_cols)
        blinds = orc.fr_random_chacha(n_blinds, 0xb00 + s).reshape(-1, 4)
        z_want, last_o = orc.permutation_product(k, values[lo:hi], sigma[lo:hi], lo, beta, gamma, blinds, last_o)
        launches, last_g = _counted(b, lambda: b.permutation_product_dev(k, [t.data_ptr() for t in dv[lo:hi]], [t.data_ptr() for t in ds[lo:hi]], lo, beta, gamma,
                                                                         blinds, last_g, dz.data_ptr()))
        assert np.array_equal(_down(dz), z_want), "set %d" % s
        assert np.array_equal(last_g, last_o.reshape(4)), "set %d" % s
        assert launches == _fraction_product_launches(G, n)


# ---- six-step NTT ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=8)
def _ntt_case(orc, k):
    a = orc.fr_random_chacha(1 << k, 0x5eed0400 + k)
    w = pyref.omega(k)
    omega, omega_inv = orc.fr([w])[0], orc.fr([pow(w, -1, R)])[0]
    fwd = orc.best_fft(a, omega, k)
    return a, omega, omega_inv, fwd, orc.best_fft(fwd, omega_inv, k)


@pytest.mark.parametrize("k", range(16, 24))
@pytest.mark.parametrize("G", [2, 4, 8])
def test_six_step_ntt(orc, G, k):
    """a host-buffer NTT of 2^k points on G devices: forward and inverse equal the oracle, and a transform launches each
    device's passes plus one gather kernel per device (the one-device path launches the passes once)"""
    b = _ctx(G)
    a, omega, omega_inv, fwd, back = _ntt_case(orc, k)
    assert np.array_equal(b.best_fft(a, omega, k), fwd)
    assert np.array_equal(b.best_fft(fwd, omega_inv, k), back)
    launches, _ = _counted(b, lambda: b.best_fft(a, omega, k))
    assert launches == G * _npass(k) + G


@pytest.mark.parametrize("G", [2, 8])
def test_six_step_domain_ops(orc, G):
    """the host-buffer EvaluationDomain ops on G devices with their fused options: coeff_to_extended's n_in zero padding and
    zeta pre-scale, extended_to_coeff's n_out truncation and post-scale, lagrange_to_coeff's 1/n post-scale"""
    from spectre_b200 import halo2
    b = _ctx(G)
    for j, k in ((4, 16), (3, 18), (9, 16)):
        d, od = halo2.EvaluationDomain(b, j, k), orc.Domain(j, k)
        a = orc.fr_random_chacha(1 << k, 0xc00 + k)
        coeff = d.lagrange_to_coeff(a)
        assert np.array_equal(coeff, od.lagrange_to_coeff(a)), (j, k)
        assert np.array_equal(d.coeff_to_lagrange(coeff), a), (j, k)
        ext = d.coeff_to_extended(coeff)
        assert np.array_equal(ext, od.coeff_to_extended(coeff)), (j, k)
        launches, again = _counted(b, lambda: d.coeff_to_extended(coeff))
        assert np.array_equal(again, ext) and launches == G * _npass(d.extended_k) + G, (j, k)
        e = orc.fr_random_chacha(1 << d.extended_k, 0xd00 + k)
        assert np.array_equal(d.extended_to_coeff(e), od.extended_to_coeff(e)), (j, k)
        del d


def test_six_step_ntt_over_32_devices_takes_the_copy_all_to_all(orc):
    """above 16 devices the all-to-all is cudaMemcpy2DAsync, not the gather kernel: 32 entries at k = 20 (where the six-step
    split applies: first digit 10 > log2 32, remaining 10 > 6) launch only the passes"""
    from spectre_b200 import halo2
    k, G = 20, 32
    a, omega, omega_inv, fwd, back = _ntt_case(orc, k)
    b = halo2.Backend([0] * G)
    try:
        assert np.array_equal(b.best_fft(a, omega, k), fwd)
        assert np.array_equal(b.best_fft(fwd, omega_inv, k), back)
        launches, _ = _counted(b, lambda: b.best_fft(a, omega, k))
        assert launches == G * _npass(k)
    finally:
        b.release_workspace()
        b.close()


# ---- sharded MSM -------------------------------------------------------------------------------------------------------
MSM_K = 10


@functools.lru_cache(maxsize=1)
def _one_device_params(be, orc):
    from spectre_b200.halo2 import ParamsKZG
    return ParamsKZG.setup(be, MSM_K, orc.srs_tau())


@functools.lru_cache(maxsize=8)
def _aliased_params(G, orc, tables):
    from spectre_b200.halo2 import ParamsKZG
    p = ParamsKZG.setup(_ctx(G), MSM_K, orc.srs_tau())
    return p.precompute() if tables else p


def _msm_lengths(G):
    """1, fewer points than shards (the later shards get none), one below and one above every shard boundary, and all"""
    n = 1 << MSM_K
    starts = [n * i // G for i in range(1, G)]
    return sorted({1, G - 1 if G > 2 else 1, n} | {s - 1 for s in starts} | {s + 1 for s in starts})


@pytest.mark.parametrize("tables", [False, True], ids=["plain", "tables"])
@pytest.mark.parametrize("G", GS)
def test_sharded_msm(be, orc, G, tables):
    """commit and commit_lagrange on an SRS sharded over G devices, from host and device-resident scalars (the shards after the
    first receive theirs by peer copy), against the known-secret commitment and the one-device result. Without tables each
    non-empty shard launches what the same MSM of its length launches on one device."""
    from spectre_b200.halo2 import BASIS_G, BASIS_G_LAGRANGE
    params, one = _aliased_params(G, orc, tables), _one_device_params(be, orc)
    b, n_srs = params.be, 1 << MSM_K
    for n in _msm_lengths(G):
        sc = orc.fr_random_chacha(n, 0xe00 + n)
        want = orc.commit_known_tau(sc)
        launches, got = _counted(b, lambda: params.commit(sc))
        assert np.array_equal(orc.g1_to_affine(got), want), n
        assert np.array_equal(orc.g1_to_affine(params.commit_lagrange(sc)), orc.commit_lagrange_known_tau(MSM_K, sc)), n
        ds = _up(sc)
        assert np.array_equal(orc.g1_to_affine(params.commit_dev(BASIS_G, ds.data_ptr(), n)), want), n
        assert np.array_equal(orc.g1_to_affine(params.commit_dev(BASIS_G_LAGRANGE, ds.data_ptr(), n)), orc.g1_to_affine(one.commit_lagrange(sc))), n
        if not tables:
            shards = [(n_srs * i // G, n_srs * (i + 1) // G) for i in range(G)]
            per_shard = sum(_counted(one.be, lambda: one.commit(sc[lo:min(hi, n)]))[0] for lo, hi in shards if lo < n)
            assert launches == per_shard, n


@pytest.mark.parametrize("G", GS)
def test_sharded_msm_batch_reuses_lanes(be, orc, G):
    """a batch of 5 commitments through the batch API, host and device scalars: the lanes of every shard are reused"""
    from spectre_b200.halo2 import BASIS_G
    params = _aliased_params(G, orc, False)
    n = (1 << MSM_K) - 3
    polys = [orc.fr_random_chacha(n, 0xf00 + i) for i in range(5)]
    want = [orc.commit_known_tau(p) for p in polys]
    got = params.commit_batch(BASIS_G, polys)
    assert all(np.array_equal(orc.g1_to_affine(g), w) for g, w in zip(got, want))
    d = [_up(p) for p in polys]
    got = params.commit_batch_dev(BASIS_G, [t.data_ptr() for t in d], n)
    assert all(np.array_equal(orc.g1_to_affine(g), w) for g, w in zip(got, want))


# ---- quotient row shards -----------------------------------------------------------------------------------------------
QUOTIENT_SIZES = [1 << 12, 1 << 17]
ROT_SCALE = 4


@functools.lru_cache(maxsize=2)
def _columns(E):
    host = [_residues(E, (E << 4) + i) for i in range(24)]
    return host, [_up(a) for a in host]


def _both(be, G, run, E):
    """run(b, d_out) on the one-device context and on the G-aliased one, on the same input column"""
    host, dev = _columns(E)
    outs = []
    for b in (be, _ctx(G)):
        dv = dev[-1].clone()
        import torch
        torch.cuda.synchronize()
        run(b, dv)
        outs.append(_down(dv))
    return outs


@pytest.mark.parametrize("E", QUOTIENT_SIZES)
@pytest.mark.parametrize("G", GS)
def test_graph_evaluate_by_row_range(be, orc, shard_small, G, E):
    """a random 150-step program reading rotations -(bf+1)..3 (so reads cross range boundaries and wrap) on G row ranges,
    against the oracle and the one-device pass"""
    prog, ncalc, constants, rotations, (nf, na, ni), challenges = _graph_case(orc, "random150")
    assert min(rotations) < -1 and max(rotations) == 3
    host, dev = _columns(E)
    bgty = _residues(4, 7)
    want = orc.graph_evaluate(prog, ncalc, ncalc, constants, rotations, host[0:nf], host[nf:nf + na], host[nf + na:nf + na + ni], challenges, bgty,
                              host[-1], ROT_SCALE)
    ptrs = lambda ts: [t.data_ptr() for t in ts]
    one, many = _both(be, G, lambda b, dv: b.graph_evaluate_dev(prog, ncalc, ncalc, constants, rotations, ptrs(dev[0:nf]), ptrs(dev[nf:nf + na]),
                                                               ptrs(dev[nf + na:nf + na + ni]), challenges, *bgty, dv.data_ptr(), E, ROT_SCALE), E)
    assert np.array_equal(one, want)
    assert np.array_equal(many, want)


@pytest.mark.parametrize("E", QUOTIENT_SIZES)
@pytest.mark.parametrize("G", GS)
def test_permutation_and_lookup_constraints_by_row_range(be, orc, shard_small, G, E):
    """permutation_constraints_dev (3 sets of 2 columns, last rotation -(bf+1)), its coset form on one n-row part, and
    lookup_constraints_dev on G row ranges equal the one-device passes"""
    from spectre_b200 import circuits
    host, dev = _columns(E)
    last_rotation = -(circuits.halo2lib_shape().blinding_factors() + 1)
    od = orc.Domain(4, E.bit_length() - 3)
    beta, gamma, y = _residues(3, 8)
    z, cv, sg, rest = dev[0:3], dev[3:8], dev[8:13], [t.data_ptr() for t in dev[13:16]]
    ptrs = lambda ts: [t.data_ptr() for t in ts]
    perm = lambda b, dv: b.permutation_constraints_dev(dv.data_ptr(), E, ROT_SCALE, last_rotation, 2, ptrs(z), ptrs(cv), ptrs(sg), *rest, beta, gamma, y,
                                                       od.extended_omega)
    one, many = _both(be, G, perm, E)
    assert np.array_equal(one, orc.permutation_constraints(host[-1], ROT_SCALE, last_rotation, 2, host[0:3], host[3:8], host[8:13], *host[13:16], beta,
                                                           gamma, y, od.extended_omega))
    assert np.array_equal(many, one)
    # a coset part: X = zeta * extended_omega^part * omega^row, rows in steps of one
    part = 3
    g = orc.fr([pyref.ZETA * pow(orc.fr_ints(od.extended_omega)[0], part, R) % R])[0]
    coset = lambda b, dv: b.permutation_constraints_coset_dev(dv.data_ptr(), E, 1, last_rotation, 2, ptrs(z), ptrs(cv), ptrs(sg), *rest, beta, gamma, y, g,
                                                              orc.fr([pyref.omega(E.bit_length() - 1)])[0])
    one, many = _both(be, G, coset, E)
    assert np.array_equal(many, one)
    look = lambda b, dv: b.lookup_constraints_dev(dv.data_ptr(), E, ROT_SCALE, *[t.data_ptr() for t in dev[16:23]], beta, gamma, y)
    one, many = _both(be, G, look, E)
    assert np.array_equal(one, orc.lookup_constraints(host[-1], ROT_SCALE, *host[16:23], beta, gamma, y))
    assert np.array_equal(many, one)


# ---- batch NTTs by polynomial ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", GS)
def test_batch_ntts_by_polynomial(be, orc, shard_small, G):
    """lagrange_to_coeff_batch_dev, coeff_to_extended_batch_dev and coeff_to_extended_part_batch_dev (every part) with 1, G - 1,
    G and 2G + 1 polynomials spread over G devices, against the one-device calls. Polynomial i runs the same passes on whichever
    device takes it, so a launch count cannot tell the two paths apart; the values must be the same."""
    import torch
    from spectre_b200 import halo2
    j, k = 4, 10
    for count in sorted({1, G - 1, G, 2 * G + 1}):
        polys = [orc.fr_random_chacha(1 << k, 0x1000 + 16 * count + i) for i in range(count)]
        results = []
        for b in (be, _ctx(G)):
            d = halo2.EvaluationDomain(b, j, k)
            R_ = 1 << (d.extended_k - k)
            ins = [_up(p) for p in polys]
            d.lagrange_to_coeff_batch_dev([t.data_ptr() for t in ins])
            exts = [torch.empty((1 << d.extended_k, 4), dtype=torch.int64, device="cuda") for _ in polys]
            d.coeff_to_extended_batch_dev([t.data_ptr() for t in ins], [t.data_ptr() for t in exts])
            parts = []
            for part in range(R_):
                outs = [torch.empty((1 << k, 4), dtype=torch.int64, device="cuda") for _ in polys]
                d.coeff_to_extended_part_batch_dev(part, [t.data_ptr() for t in ins], [t.data_ptr() for t in outs])
                parts.append([_down(t) for t in outs])
            results.append(([_down(t) for t in ins], [_down(t) for t in exts], parts))
            del d
        (c1, e1, p1), (cg, eg, pg) = results
        od = orc.Domain(j, k)
        assert all(np.array_equal(c, od.lagrange_to_coeff(p)) for c, p in zip(c1, polys)), count
        assert all(np.array_equal(a, b_) for a, b_ in zip(c1, cg)), count
        assert all(np.array_equal(a, b_) for a, b_ in zip(e1, eg)), count
        for part, (x, y_) in enumerate(zip(p1, pg)):
            assert all(np.array_equal(a, e[part::len(p1)]) for a, e in zip(x, e1)), (count, part)
            assert all(np.array_equal(a, b_) for a, b_ in zip(x, y_)), (count, part)


# ---- whole proofs ------------------------------------------------------------------------------------------------------
def _halo2lib_case():
    from spectre_b200 import circuits
    k, instances = 12, [3, 1, 4]
    cs = circuits.halo2lib_shape(4, 1)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=5, groups=200, num_gate_advice=4, num_lookup_advice=1)
    return k, instances, cs, fixed, adv, copies


def _proof(b, orc, cosets):
    from spectre_b200 import halo2, plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    k, instances, cs, fixed, adv, copies = _halo2lib_case()
    E = plonk.DeviceEngine(b, halo2.ParamsKZG.setup(b, k, orc.srs_tau()).precompute(), k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, cosets=cosets)
    return pk, plonk.create_proof(E, pk, [instances], adv, SeededRng(5), EvmTranscriptWrite(pk.vk_digest))


@functools.lru_cache(maxsize=1)
def _one_device_proof(be, orc):
    return _proof(be, orc, "resident")[1]


@pytest.mark.parametrize("cosets", ["resident", "on_demand", "per_part"])
@pytest.mark.parametrize("G", GS)
def test_halo2lib_proof_on_aliased_devices(be, orc, shard_small, G, cosets):
    """the halo2lib shape at k = 12 with every multi-device path on (sharded MSMs, row-range quotient passes and grand
    products, batch NTTs by polynomial): byte-identical to the one-device proof, and accepted by the verifier"""
    from spectre_b200 import plonk
    from tests import plonk_verifier
    assert cosets in plonk.COSETS_MODES
    pk, proof = _proof(_ctx(G), orc, cosets)
    assert proof == _one_device_proof(be, orc)
    k, instances, cs = _halo2lib_case()[:3]
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    assert plonk_verifier.verify(cs, k, pk.vk_digest, pk.fixed_commitments, pk.sigma_commitments, [instances], proof, tau)


@pytest.mark.slow
def test_k23_fixture_on_two_aliased_devices(be, orc):
    """the K = 23 aggregation proof of tests/golden/aggregation_k23_proof.json, regenerated byte for byte on [0, 0] at the
    default sharding thresholds"""
    import json
    import os
    import torch
    from spectre_b200 import circuits, halo2, plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    for b in list(_contexts.values()):
        b.release_workspace()
    be.release_workspace()
    with open(os.path.join(os.path.dirname(__file__), "golden", "aggregation_k23_proof.json")) as f:
        fx = json.load(f)
    k = fx["k"]
    instances = [int(v, 16) for v in fx["instances"]]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, fx["lookup_bits"], fx["groups"], seed=fx["seed"])
    b = _ctx(2)
    params = halo2.ParamsKZG.setup(b, k, orc.srs_tau()).precompute()
    E = plonk.DeviceEngine(b, params, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=int(fx["vk_digest"]))
    proof = plonk.create_proof(E, pk, [instances], [adv], SeededRng(fx["seed"]), EvmTranscriptWrite(pk.vk_digest))
    free, total = torch.cuda.mem_get_info(0)
    print("K = 23 on [0, 0]: %.2f GiB of device memory in use after the proof" % ((total - free) / 2 ** 30))
    assert proof.hex() == fx["proof"]
    del E, pk, params
    b.release_workspace()
