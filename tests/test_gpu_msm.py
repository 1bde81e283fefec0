"""GPU parity of best_multiexp / ParamsKZG::commit* through the C ABI against the CPU oracle (bit-exact affine
equality) and against the reference-owned known-answer vectors."""
import json
import os

import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be, device_lists  # noqa: F401

pytestmark = pytest.mark.gpu


def affine_of(orc, jac):
    return orc.g1_to_affine(jac)


@pytest.fixture(scope="module")
def points(orc):
    return orc.g1_fixed_base_mul(orc.fr_random_chacha(1 << 14, 0x5eed0002))


def test_fixed_base_mul_matches_oracle(be, orc):
    sc = orc.fr_random_chacha(257, 11)
    sc[0] = 0
    sc[1] = orc.fr([1])[0]
    sc[2] = orc.fr([pyref.R_MOD - 1])[0]
    assert np.array_equal(be.g1_fixed_base_mul(sc), orc.g1_fixed_base_mul(sc))


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 255, 1000, 4096, 1 << 14])
def test_best_multiexp_uniform(be, orc, points, n):
    sc = orc.fr_random_chacha(n, 0x5eed0003 + n)
    got = affine_of(orc, be.best_multiexp(sc, points[:n]))
    want = affine_of(orc, orc.best_multiexp(sc, points[:n]))
    assert np.array_equal(got, want)


def test_best_multiexp_empty(be, orc):
    out = be.best_multiexp(np.zeros((0, 4), dtype=np.uint64), np.zeros((0, 8), dtype=np.uint64))
    assert not out[8:].any()  # z = 0: identity


def test_length_mismatch_panics(be, orc, points):
    with pytest.raises(AssertionError):
        be.best_multiexp(orc.fr([1, 2, 3]), points[:2])


@pytest.mark.parametrize("label", ["all_zero", "all_one", "all_minus_one", "single_nonzero", "dup_bases", "identity_bases", "cancel", "witness_like"])
def test_edge_distributions(be, orc, points, label):
    n = 5000
    bases = points[:n].copy()
    rng = np.random.default_rng(5)
    if label == "all_zero":
        ks = [0] * n
    elif label == "all_one":
        ks = [1] * n
    elif label == "all_minus_one":
        ks = [pyref.R_MOD - 1] * n
    elif label == "single_nonzero":
        ks = [0] * n; ks[1234] = 0xdeadbeefcafebabe1234567
    elif label == "dup_bases":
        ks = [int(x) for x in rng.integers(1, 1 << 62, n)]
        bases[:] = bases[0]
    elif label == "identity_bases":
        ks = [int(x) for x in rng.integers(1, 1 << 62, n)]
        bases[::3] = 0
    elif label == "cancel":
        ks = [5] * n
        half = n // 2
        bases[half:2 * half] = bases[:half]
        bases[half:2 * half, 4:] = orc.fq([(-y) % pyref.P_MOD for y in orc.fq_ints(bases[:half, 4:])])
    else:
        ks = []
        for i in range(n):
            u = rng.random()
            ks.append(0 if u < 0.7 else int(rng.integers(0, 1 << 16)) if u < 0.9 else int(rng.integers(0, 1 << 62)) ** 2 % (1 << 104) if u < 0.99 else int(rng.integers(1, 1 << 62)) ** 4 % pyref.R_MOD)
    sc = orc.fr(ks)
    got = affine_of(orc, be.best_multiexp(sc, bases))
    want = affine_of(orc, orc.best_multiexp(sc, bases))
    assert np.array_equal(got, want), label
    if label == "all_zero":
        assert not got.any()


def test_giant_bucket_block_path(be, orc, points):
    """2^14 equal scalars -> one bucket chain far longer than the stitch cap (block-wide tree path)."""
    n = 1 << 14
    sc = np.repeat(orc.fr([1]), n, axis=0)
    got = affine_of(orc, be.best_multiexp(sc, points[:n]))
    want = affine_of(orc, orc.best_multiexp(sc, points[:n]))
    assert np.array_equal(got, want)


def test_huge_chain_grid_path(be, orc):
    """2^18 equal scalars: one bucket chain of 8192 chunk pieces (> 4096) -> the grid-wide huge-chain kernels; also a
    0/1 column. Expected values by group arithmetic on the oracle: sum of all points / of the selected points."""
    k = 18
    n = 1 << k
    pts = be.g1_fixed_base_mul(orc.fr_random_chacha(n, 0x5eed0042))
    assert np.array_equal(pts[:64], orc.g1_fixed_base_mul(orc.fr_random_chacha(n, 0x5eed0042)[:64]))
    ones = np.repeat(orc.fr([1]), n, axis=0)
    total = be.best_multiexp(ones, pts)
    # the same sum through a different schedule: random scalars r and 1 - r
    r = orc.fr_random_chacha(n, 7)
    one_minus_r = be.vec_axpy(ones, orc.fr([pyref.R_MOD - 1])[0], r)
    alt = orc.g1_add(be.best_multiexp(r, pts), be.best_multiexp(one_minus_r, pts))
    assert np.array_equal(affine_of(orc, total), orc.g1_to_affine(alt))
    bits = np.zeros((n, 4), dtype=np.uint64)
    sel = np.random.default_rng(1).random(n) < 0.5
    bits[sel] = orc.fr([1])[0]
    masked = r.copy(); masked[~sel] = 0
    compl = be.vec_axpy(bits, orc.fr([pyref.R_MOD - 1])[0], masked)       # bits - masked r
    alt = orc.g1_add(be.best_multiexp(masked, pts), be.best_multiexp(compl, pts))
    assert np.array_equal(affine_of(orc, be.best_multiexp(bits, pts)), orc.g1_to_affine(alt))
    # and directly against the CPU port on a prefix large enough to take the huge path with a small window choice
    m = 1 << 17
    assert np.array_equal(affine_of(orc, be.best_multiexp(ones[:m], pts[:m])), affine_of(orc, orc.best_multiexp(ones[:m], pts[:m])))


def test_params_kzg_setup_and_commit_seed0(be, orc):
    """ParamsKZG::setup on the device with the seed-0 secret reproduces the oracle's (KAT-pinned) SRS, and
    commit / commit_lagrange agree with both best_multiexp and the O(n) known-tau shortcut."""
    from spectre_b200.halo2 import ParamsKZG, BASIS_G, BASIS_G_LAGRANGE
    k = 10
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    assert np.array_equal(params.get_g(basis=BASIS_G), orc.srs_g(k, 0, 1 << k))
    assert np.array_equal(params.get_g(basis=BASIS_G_LAGRANGE), orc.srs_g_lagrange(k, 0, 1 << k))
    poly = orc.fr_random_chacha(1 << k, 321)
    assert np.array_equal(affine_of(orc, params.commit(poly)), orc.commit_known_tau(poly))
    assert np.array_equal(affine_of(orc, params.commit_lagrange(poly)), orc.commit_lagrange_known_tau(k, poly))
    short = poly[:100]  # commit of a shorter polynomial uses g[..len]
    assert np.array_equal(affine_of(orc, params.commit(short)), orc.commit_known_tau(short))


@pytest.mark.parametrize("k,k2", [(10, 7), (12, 12), (9, 0)])
def test_params_kzg_downsize(be, orc, k, k2):
    """ParamsKZG::downsize(k2): g truncated, g_lagrange recomputed by the group inverse DFT on the device -- must equal the
    seed-0 SRS of the smaller domain (the derivation pinned by the verifier contracts), and commitments through it the
    known-tau values. The original handle is untouched."""
    from spectre_b200.halo2 import ParamsKZG, BASIS_G, BASIS_G_LAGRANGE
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    small = params.downsize(k2)
    n2 = 1 << k2
    assert np.array_equal(small.get_g(basis=BASIS_G), orc.srs_g(k2, 0, n2))
    assert np.array_equal(small.get_g(basis=BASIS_G_LAGRANGE), orc.srs_g_lagrange(k2, 0, n2))
    poly = orc.fr_random_chacha(n2, 77)
    assert np.array_equal(affine_of(orc, small.commit_lagrange(poly)), orc.commit_lagrange_known_tau(k2, poly))
    assert np.array_equal(params.get_g(basis=BASIS_G_LAGRANGE), orc.srs_g_lagrange(k, 0, 1 << k))
    with pytest.raises(Exception):
        params.downsize(k + 1)


def test_two_contexts_prove_concurrently_on_one_device(orc):
    """Spectre's RPC `--concurrency N` (prover/src/prover.rs:114): one context per concurrent proof on the same GPU, sharing
    nothing but the device. Two threads prove at the same time; both proofs are byte-identical to the sequential ones."""
    import threading
    from spectre_b200 import circuits, halo2, plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    k, instances = 11, [3, 1, 4]
    cs = circuits.halo2lib_shape(4, 1)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=5, groups=100, num_gate_advice=4, num_lookup_advice=1)
    ctxs = [halo2.Backend([0]) for _ in range(2)]
    try:
        engines, keys = [], []
        for b in ctxs:
            E = plonk.DeviceEngine(b, halo2.ParamsKZG.setup(b, k, orc.srs_tau()), k, cs.degree())
            engines.append(E); keys.append(plonk.keygen(E, cs, k, fixed, copies, vk_digest=99))
        want = [plonk.create_proof(E, pk, [instances], adv, SeededRng(5 + i), EvmTranscriptWrite(pk.vk_digest)) for i, (E, pk) in enumerate(zip(engines, keys))]
        got, errs = [None, None], []

        def work(i):
            try:
                for _ in range(3):
                    got[i] = plonk.create_proof(engines[i], keys[i], [instances], adv, SeededRng(5 + i), EvmTranscriptWrite(keys[i].vk_digest))
            except Exception as e:   # noqa: BLE001
                errs.append(e)
        ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
        [t.start() for t in ts]; [t.join() for t in ts]
        assert not errs, errs
        assert got == want
    finally:
        for b in ctxs:
            b.close()


def test_reference_kat_range_table_k23(be, orc, kats):
    """The reference's own pinned number: commit_lagrange(range table 0..2^19) under the seed-0 SRS at K=23 equals
    the fixed-column commitment in contracts/snark-verifiers/sync_step_verifier.sol:1048-1049. Only the first 2^19
    Lagrange points matter (the rest multiply zeros), so they are generated by the oracle and uploaded."""
    kat = kats["range_table_commit_k23_bits19"]
    n_used = 1 << kat["lookup_bits"]
    bases = orc.srs_g_lagrange(kat["k"], 0, n_used)
    coeffs = orc.fr_seq(n_used)
    got = orc.affine_ints(affine_of(orc, be.best_multiexp(coeffs, bases)))[0]
    assert list(got) == [int(v, 16) for v in kat["xy"]]


@pytest.mark.parametrize("k", [18, 20])
def test_large_msm_known_tau(be, orc, k):
    """BASELINE config 2 size (2^20): SRS generated on the device, result checked with the known-tau oracle
    (independent of any MSM code) and a size-independent linearity property."""
    from spectre_b200.halo2 import ParamsKZG
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    n = 1 << k
    a = orc.fr_random_chacha(n, 0x5eed0003)
    ca = affine_of(orc, params.commit(a))
    assert np.array_equal(ca, orc.commit_known_tau(a))
    cl = affine_of(orc, params.commit_lagrange(a))
    assert np.array_equal(cl, orc.commit_lagrange_known_tau(k, a))
    # linearity: commit(a) + commit(b) == commit(a + b)
    b = orc.fr_random_chacha(n, 0x5eed0004)
    ab = be.vec_axpy(a, orc.fr([1])[0], b)
    lhs = orc.g1_to_affine(orc.g1_add(params.commit(a), params.commit(b)))
    assert np.array_equal(lhs, affine_of(orc, params.commit(ab)))


def test_precomputed_tables_and_batch(be, orc):
    """spb_srs_precompute changes only the schedule (one bucket set, wider window): every commitment must be
    identical to the table-free path and to the oracle; the two-lane batch API returns out[i] for scalars[i]."""
    from spectre_b200.halo2 import ParamsKZG, BASIS_G, BASIS_G_LAGRANGE
    k = 12
    n = 1 << k
    g = orc.srs_g(k, 0, n); gl = orc.srs_g_lagrange(k, 0, n)
    plain = ParamsKZG.from_parts(be, k, g, gl)
    tabled = ParamsKZG.from_parts(be, k, g, gl).precompute()
    polys = [orc.fr_random_chacha(n, 7000 + i) for i in range(5)]
    polys[1][::2] = 0
    polys[2][:] = orc.fr([1])[0]                    # giant bucket through the table path
    polys[3][:] = orc.fr([pyref.R_MOD - 1])[0]      # every window non-zero, all digits negative-capable
    want = [orc.g1_to_affine(orc.best_multiexp(p, gl)) for p in polys]
    for p, w in zip(polys, want):
        assert np.array_equal(affine_of(orc, plain.commit_lagrange(p)), w)
        assert np.array_equal(affine_of(orc, tabled.commit_lagrange(p)), w)
    batch = tabled.commit_batch(BASIS_G_LAGRANGE, polys)
    for row, w in zip(batch, want):
        assert np.array_equal(affine_of(orc, row), w)
    batch = plain.commit_batch(BASIS_G_LAGRANGE, polys[:1])   # count = 1 edge
    assert np.array_equal(affine_of(orc, batch[0]), want[0])
    # shorter polynomial against the table: uses g[..len] of every table row
    short = polys[0][:777]
    assert np.array_equal(affine_of(orc, tabled.commit(short)), orc.commit_known_tau(short))
    assert np.array_equal(affine_of(orc, plain.commit(short)), orc.commit_known_tau(short))


def test_large_msm_tables_known_tau(be, orc):
    """2^20 with tables (the bench configuration): known-tau check, independent of any MSM code."""
    from spectre_b200.halo2 import ParamsKZG
    k = 20
    params = ParamsKZG.setup(be, k, orc.srs_tau()).precompute()
    a = orc.fr_random_chacha(1 << k, 0x5eed0007)
    assert np.array_equal(affine_of(orc, params.commit(a)), orc.commit_known_tau(a))
    assert np.array_equal(affine_of(orc, params.commit_lagrange(a)), orc.commit_lagrange_known_tau(k, a))


@pytest.mark.parametrize("ids", device_lists())
def test_multi_device_context(orc, ids):
    """n_dev > 1 in one context: SRS sharded by point range, partial sums folded on the host."""
    from spectre_b200 import halo2
    be2 = halo2.Backend(ids)
    k = 11
    n = 1 << k
    gl = orc.srs_g_lagrange(k, 0, n)
    params = halo2.ParamsKZG.from_parts(be2, k, g_lagrange=gl)
    p = orc.fr_random_chacha(n, 4242)
    want = orc.g1_to_affine(orc.best_multiexp(p, gl))
    assert np.array_equal(orc.g1_to_affine(params.commit_lagrange(p)), want)
    params.precompute()
    assert np.array_equal(orc.g1_to_affine(params.commit_lagrange(p)), want)
    assert np.array_equal(orc.g1_to_affine(be2.best_multiexp(p, gl)), want)
    be2.close()


def test_full_size_k23_known_tau_and_linearity(be, orc):
    """BASELINE full size (aggregation K = 23): SRS and window tables generated on the device; commit checked with the
    O(n) known-tau oracle (independent of every MSM code path) and with linearity commit(a)+commit(b) == commit(a+b)."""
    import torch
    from spectre_b200.halo2 import ParamsKZG, BASIS_G_LAGRANGE
    k = 23
    n = 1 << k
    params = ParamsKZG.setup(be, k, orc.srs_tau()).precompute()
    a = orc.fr_random_chacha(n, 0x5eed0023)
    ca = params.commit(a)
    assert np.array_equal(affine_of(orc, ca), orc.commit_known_tau(a))
    b = orc.fr_random_chacha(n, 0x5eed0024)
    da, db = (torch.from_numpy(x.view(np.int64)).cuda() for x in (a, b))
    be.lib.spb_vec_axpy_dev  # exported
    one = orc.fr([1])[0]
    cb = params.commit_dev(0, db.data_ptr(), n)
    be.check(be.lib.spb_vec_axpy_dev(be.ctx, __import__("ctypes").c_void_p(da.data_ptr()), one.ctypes.data_as(__import__("ctypes").c_void_p),
                                     __import__("ctypes").c_void_p(db.data_ptr()), __import__("ctypes").c_size_t(n)), "spb_vec_axpy_dev")
    cab = params.commit_dev(0, da.data_ptr(), n)
    assert np.array_equal(orc.g1_to_affine(orc.g1_add(ca, cb)), affine_of(orc, cab))
    # the reference-owned K = 23 known answer through the resident Lagrange basis WITH tables
    import json, os
    with open(os.path.join(os.path.dirname(__file__), "golden", "verifier_kats.json")) as f:
        kat = json.load(f)["range_table_commit_k23_bits19"]
    table = np.zeros((n, 4), dtype=np.uint64)
    table[: 1 << kat["lookup_bits"]] = orc.fr_seq(1 << kat["lookup_bits"])
    got = orc.affine_ints(affine_of(orc, params.commit_lagrange(table)))[0]
    assert list(got) == [int(v, 16) for v in kat["xy"]]


def test_params_file_read_write_roundtrip(be, orc, tmp_path):
    """ParamsKZG::read of a gen_srs-style params file (written by the oracle in SerdeFormat::RawBytes), commit through
    it, write it back byte-identically."""
    from spectre_b200.halo2 import ParamsKZG, BASIS_G, BASIS_G_LAGRANGE
    k = 9
    src = str(tmp_path / ("kzg_bn254_%d.srs" % k))
    g2, s_g2 = orc.write_params_file(src, k)
    params = ParamsKZG.read(be, src)
    assert params.k == k
    assert np.array_equal(params.get_g(basis=BASIS_G), orc.srs_g(k, 0, 1 << k))
    assert np.array_equal(params.get_g(basis=BASIS_G_LAGRANGE), orc.srs_g_lagrange(k, 0, 1 << k))
    got_g2, got_s = params.get_g2()
    assert np.array_equal(got_g2.reshape(4, 4), g2) and np.array_equal(got_s.reshape(4, 4), s_g2)
    poly = orc.fr_random_chacha(1 << k, 5)
    assert np.array_equal(affine_of(orc, params.commit_lagrange(poly)), orc.commit_lagrange_known_tau(k, poly))
    dst = str(tmp_path / "copy.srs")
    params.write(dst)
    assert open(src, "rb").read() == open(dst, "rb").read()
    with pytest.raises(Exception):
        ParamsKZG.read(be, str(tmp_path / "missing.srs"))


@pytest.mark.parametrize("label", ["uniform", "all_minus_one", "witness_like", "zeros_and_ones", "pairs"])
def test_counting_sort_groups_repeated_digits_only_when_neighbours_repeat(be, orc, points, label):
    """The histogram / scatter kernels serve equal digits of a warp with one atomic only when neighbouring lanes repeat
    (msm_warp_peers: the MATCH.ANY grouping is skipped otherwise); duplicates that are NOT neighbours take their own atomics.
    All of these columns -- uniform, constant, witness-like, 0/1, and values repeated at distance 2 -- must give the oracle's
    points through best_multiexp (W bucket sets) and the tabled commit_lagrange (one bucket set), ragged lengths included."""
    from spectre_b200.halo2 import ParamsKZG
    k = 13
    n = 1 << k
    rng = np.random.default_rng(17)
    if label == "uniform":
        sc = orc.fr_random_chacha(n, 0xb1)
    elif label == "all_minus_one":
        sc = orc.fr([pyref.R_MOD - 1] * n)
    elif label == "zeros_and_ones":
        sc = orc.fr([int(x) for x in rng.integers(0, 2, n)])
    elif label == "pairs":                                          # a, b, a, b, ... : every digit repeated at distance 2, never adjacent
        sc = orc.fr_random_chacha(n, 0xb2)
        sc[2::4] = sc[0::4]; sc[3::4] = sc[1::4]
    else:
        ks = []
        for i in range(n):
            u = rng.random()
            ks.append(0 if u < 0.7 else int(rng.integers(0, 1 << 16)) if u < 0.9 else int(rng.integers(0, 1 << 62)) ** 2 % (1 << 104) if u < 0.99 else int(rng.integers(1, 1 << 62)) ** 4 % pyref.R_MOD)
        sc = orc.fr(ks)
    want = affine_of(orc, orc.best_multiexp(sc, points[:n]))
    assert np.array_equal(affine_of(orc, be.best_multiexp(sc, points[:n])), want)
    for m in (n - 1, 777):
        assert np.array_equal(affine_of(orc, be.best_multiexp(sc[:m], points[:m])), affine_of(orc, orc.best_multiexp(sc[:m], points[:m]))), m
    tabled = ParamsKZG.from_parts(be, k, g_lagrange=points[:n]).precompute()
    assert np.array_equal(affine_of(orc, tabled.commit_lagrange(sc)), want)


@pytest.mark.parametrize("n", [1, 1000, 5000, (1 << 13) + 17])
def test_resident_bases_of_any_length(be, orc, points, n):
    """spb_bases_upload: bases of any length stay resident, spb_msm against them is best_multiexp without the per-call upload of
    spb_msm_raw -- same points, with and without window tables, also for a prefix of the bases."""
    from spectre_b200.halo2 import ParamsKZG
    sc = orc.fr_random_chacha(n, 0xba5e + n)
    want = affine_of(orc, orc.best_multiexp(sc, points[:n]))
    res = ParamsKZG.from_bases(be, points[:n])
    assert np.array_equal(affine_of(orc, res.multiexp(sc)), want)
    assert np.array_equal(affine_of(orc, be.best_multiexp(sc, points[:n])), want)
    m = max(1, n // 3)
    assert np.array_equal(affine_of(orc, res.multiexp(sc[:m])), affine_of(orc, orc.best_multiexp(sc[:m], points[:m])))
    res.precompute()
    assert np.array_equal(affine_of(orc, res.multiexp(sc)), want)


def test_plain_bases_handle_rejects_srs_only_operations(be, orc, points, tmp_path):
    """A spb_bases_upload handle is not a 2^k SRS: downsize / write (which assume g[2^k] and g_lagrange) fail with an error text,
    more scalars than bases are refused, and a quotient pass over a size that is not a power of two is refused at the boundary."""
    import torch
    from spectre_b200.halo2 import BackendError, ParamsKZG
    res = ParamsKZG.from_bases(be, points[:1000])
    with pytest.raises(BackendError, match="plain bases"):
        res.downsize(3)
    with pytest.raises(BackendError, match="plain bases"):
        res.write(str(tmp_path / "x.srs"))
    with pytest.raises((BackendError, AssertionError)):
        res.multiexp(orc.fr_random_chacha(1001, 3))
    dev = torch.device("cuda", 0)
    z = torch.zeros((96, 4), dtype=torch.int64, device=dev)
    with pytest.raises(BackendError, match="power of two"):
        be.lookup_constraints_dev(z.data_ptr(), 96, 1, z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(),
                                  orc.fr([1])[0], orc.fr([2])[0], orc.fr([3])[0])
