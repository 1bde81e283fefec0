"""GPU parity of the argument provers (permutation / lookup grand products, weighted sums, the SHPLONK opener) through
the C ABI against the oracle's restatement of the upstream prover code. Parity unpinned vs the Rust reference (no
reference-owned vector for these rows); the SHPLONK outputs are additionally checked to be valid openings."""
import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be, device_lists  # noqa: F401

pytestmark = pytest.mark.gpu


def _dev(torch, arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("k,n_cols,chunk,n_blinds", [(4, 1, 1, 0), (8, 5, 3, 5), (12, 7, 2, 6), (14, 3, 3, 1)])
def test_permutation_product_sets_chain(be, orc, k, n_cols, chunk, n_blinds):
    import torch
    n = 1 << k
    values = [orc.fr_random_chacha(n, 100 + c) for c in range(n_cols)]
    sigma = [orc.fr_random_chacha(n, 200 + c) for c in range(n_cols)]
    values[0][3] = 0; sigma[0][5] = 0
    beta, gamma = orc.fr_random_chacha(2, 300 + k)
    dv, ds = [_dev(torch, a) for a in values], [_dev(torch, a) for a in sigma]
    dz = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    last_o = last_g = orc.fr([1])[0]
    for s, lo in enumerate(range(0, n_cols, chunk)):
        hi = min(lo + chunk, n_cols)
        blinds = orc.fr_random_chacha(n_blinds, 400 + s).reshape(-1, 4)
        z_want, last_o = orc.permutation_product(k, values[lo:hi], sigma[lo:hi], lo, beta, gamma, blinds, last_o)
        last_g = be.permutation_product_dev(k, [t.data_ptr() for t in dv[lo:hi]], [t.data_ptr() for t in ds[lo:hi]], lo, beta, gamma, blinds, last_g, dz.data_ptr())
        assert np.array_equal(_host(dz), z_want)
        assert np.array_equal(last_g, last_o.reshape(4))


def test_permutation_product_of_a_real_permutation_closes(be, orc):
    """with sigma encoding an actual permutation of equal cells the product over the usable rows returns to 1"""
    import torch
    k, n_cols = 8, 3
    n = 1 << k
    R = pyref.R_MOD
    delta = orc.fr_ints(orc.fr_delta().reshape(1, 4))[0]
    omega = pyref.omega(k)
    ident = [[pow(delta, c, R) * pow(omega, i, R) % R for i in range(n)] for c in range(n_cols)]
    vals = [[(7 * i + c) % 50 for i in range(n)] for c in range(n_cols)]           # many equal cells
    cells = {}
    for c in range(n_cols):
        for i in range(n):
            cells.setdefault(vals[c][i], []).append((c, i))
    sig = [[0] * n for _ in range(n_cols)]
    for group in cells.values():                                                    # one cycle per value class
        for a, b in zip(group, group[1:] + group[:1]):
            sig[a[0]][a[1]] = ident[b[0]][b[1]]
    values = [orc.fr(v) for v in vals]; sigma = [orc.fr(s) for s in sig]
    beta, gamma = orc.fr_random_chacha(2, 77)
    dv, ds = [_dev(torch, a) for a in values], [_dev(torch, a) for a in sigma]
    dz = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    one = orc.fr([1])[0]
    # n_blinds = 0 and a permutation over ALL rows: z[n-1] * last factor = 1, so check z[n-1] * modified[n-1] via a second set of length 0 ... simply:
    last = be.permutation_product_dev(k, [t.data_ptr() for t in dv], [t.data_ptr() for t in ds], 0, beta, gamma, np.zeros((0, 4), np.uint64), one, dz.data_ptr())
    z = _host(dz)
    z_want, _ = orc.permutation_product(k, values, sigma, 0, beta, gamma, np.zeros((0, 4), np.uint64), one)
    assert np.array_equal(z, z_want)
    # the full product over all n rows is 1: z[n-1] * num[n-1] / den[n-1] == 1
    b, g = orc.fr_ints(np.stack([beta, gamma]))
    num = den = 1
    for c in range(n_cols):
        num = num * (vals[c][n - 1] + b * ident[c][n - 1] + g) % R
        den = den * (vals[c][n - 1] + b * sig[c][n - 1] + g) % R
    assert orc.fr_ints(z[n - 1:n])[0] * num % R == den
    assert np.array_equal(last, z[n - 1])


@pytest.mark.parametrize("n,n_blinds", [(16, 0), (1 << 10, 5), (3000, 6), (1 << 15, 6)])
def test_lookup_product(be, orc, n, n_blinds):
    import torch
    arrs = [orc.fr_random_chacha(n, 500 + i) for i in range(4)]
    beta, gamma = orc.fr_random_chacha(2, 601)
    arrs[3][9] = orc.fr([-orc.fr_ints(gamma.reshape(1, 4))[0]])[0]                   # a zero denominator: batch_invert leaves 0
    blinds = orc.fr_random_chacha(n_blinds, 602).reshape(-1, 4)
    want = orc.lookup_product(*arrs, beta, gamma, blinds)
    d = [_dev(torch, a) for a in arrs]
    dz = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    be.lookup_product_dev(n, *[t.data_ptr() for t in d], beta, gamma, blinds, dz.data_ptr())
    assert np.array_equal(_host(dz), want)


def test_weighted_sum(be, orc):
    import torch
    n, count = 5000, 9
    polys = [orc.fr_random_chacha(n, 700 + i) for i in range(count)]
    w = orc.fr_random_chacha(count, 800)
    wi = orc.fr_ints(w); pi = [orc.fr_ints(p) for p in polys]
    want = orc.fr([sum(wi[j] * pi[j][i] for j in range(count)) for i in range(n)])
    d = [_dev(torch, a) for a in polys]
    out = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    be.weighted_sum_dev([t.data_ptr() for t in d], w, out.data_ptr(), n)
    assert np.array_equal(_host(out), want)


def _open_sets(orc, n, layout, seed):
    """layout: list of (point indices, number of polys) -> (sets with host polys, point array)"""
    pts = orc.fr_random_chacha(8, seed)
    sets = []
    for si, (pidx, m) in enumerate(layout):
        polys = [orc.fr_random_chacha(n, seed * 100 + si * 10 + j) for j in range(m)]
        evals = np.stack([np.stack([orc.eval_polynomial(p, pts[i]) for i in pidx]) for p in polys])
        sets.append((pts[list(pidx)], polys, evals))
    return sets


@pytest.mark.parametrize("k,layout", [(6, [((0,), 1)]), (10, [((0,), 3), ((0, 1), 2), ((0, 1, 2), 1), ((3,), 2)]), (13, [((0, 1, 2, 3, 4), 2), ((1, 5), 4)])])
def test_shplonk_prover_matches_oracle_and_opens(be, orc, k, layout):
    import torch
    from spectre_b200.halo2 import ParamsKZG
    n = 1 << k
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    sets = _open_sets(orc, n, layout, 40 + k)
    y, v, u = orc.fr_random_chacha(3, 900 + k)
    h_x = orc.shplonk_quotient(n, sets, y, v)
    final = orc.shplonk_linearisation(n, sets, y, v, u, h_x)      # raises unless L(u) == 0
    keep = [[_dev(torch, p) for p in polys] for _, polys, _ in sets]
    dsets = [(pts, [t.data_ptr() for t in dp], ev) for (pts, _, ev), dp in zip(sets, keep)]
    h_commit, handle = be.shplonk_begin_dev(params, n, dsets, y, v)
    assert np.array_equal(orc.g1_to_affine(h_commit), orc.commit_known_tau(h_x))
    got = be.shplonk_finish_dev(handle, u)
    assert np.array_equal(orc.g1_to_affine(got), orc.commit_known_tau(final))


def test_shplonk_argument_errors(be, orc):
    import torch
    from spectre_b200.halo2 import ParamsKZG, BackendError
    k = 6; n = 1 << k
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    sets = _open_sets(orc, n, [((0,), 1), ((1,), 1)], 3)
    d = [_dev(torch, st[1][0]) for st in sets]
    y, v = orc.fr_random_chacha(2, 5)
    dup = np.stack([sets[0][0][0], sets[0][0][0]])
    with pytest.raises(BackendError):                               # a point listed twice in one rotation set
        be.shplonk_begin_dev(params, n, [(dup, [d[0].data_ptr()], np.concatenate([sets[0][2], sets[0][2]], axis=1))], y, v)
    dsets = [(st[0], [t.data_ptr()], st[2]) for st, t in zip(sets, d)]
    _, handle = be.shplonk_begin_dev(params, n, dsets, y, v)
    with pytest.raises(BackendError):                               # u on an opening point outside set 0: Z_{T \ S_0}(u) = 0 has no inverse
        be.shplonk_finish_dev(handle, sets[1][0][0])


# ---- the whole driver: create_proof on the device ---------------------------------------------------------------------
def _prove_both(be, orc, cs, k, fixed, advice, copies, instances, seed):
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import OracleEngine, SeededRng
    out = []
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    for E in (plonk.DeviceEngine(be, params, k, cs.degree()), OracleEngine(k, cs.degree())):
        pk = plonk.keygen(E, cs, k, fixed, copies)
        T = EvmTranscriptWrite(pk.vk_digest)
        out.append((pk, plonk.create_proof(E, pk, [instances], advice, SeededRng(seed), T)))
    return out


@pytest.mark.parametrize("shape,k", [("aggregation", 7), ("aggregation", 11), ("wide", 8), ("wide", 12), ("halo2lib", 10)])
def test_device_proof_is_byte_identical_to_the_oracle_proof_and_verifies(be, orc, shape, k):
    from spectre_b200 import circuits as plonk_circuits
    from tests import plonk_verifier
    instances = [3, 1, 4, 1, 5]
    if shape == "aggregation":
        cs = plonk_circuits.aggregation_shape()
        fixed, adv, copies = plonk_circuits.aggregation_witness(cs, k, instances, lookup_bits=4, groups=300)
        adv = [adv]
    elif shape == "wide":
        cs = plonk_circuits.wide_shape(3)
        fixed, adv, copies = plonk_circuits.wide_witness(cs, k, instances, lookup_bits=4, groups=300)
    else:                                                       # the sync-step circuit's multi-column shape, 11 permutation sets
        cs = plonk_circuits.halo2lib_shape()
        fixed, adv, copies = plonk_circuits.halo2lib_witness(cs, k, instances, lookup_bits=5, groups=100)
    (pk_d, proof_d), (pk_o, proof_o) = _prove_both(be, orc, cs, k, fixed, adv, copies, instances, seed=100 + k)
    assert pk_d.fixed_commitments == pk_o.fixed_commitments and pk_d.sigma_commitments == pk_o.sigma_commitments
    assert proof_d == proof_o
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    assert plonk_verifier.verify(cs, k, pk_d.vk_digest, pk_d.fixed_commitments, pk_d.sigma_commitments, [instances], proof_d, tau)


def test_random_polynomial_drawn_on_the_device_gives_the_oracle_proof(be, orc):
    """plonk.DeviceBulkRng: the vanishing argument's random polynomial comes from spb_fr_random_chacha_dev (never on the host);
    the oracle engine draws the same ChaCha20 stream on the CPU, so the proofs are byte-identical and verify."""
    from spectre_b200 import circuits as plonk_circuits, plonk
    from spectre_b200.halo2 import ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests import plonk_verifier
    from tests.plonk_oracle_engine import OracleEngine, SeededRng
    k, instances = 9, [2, 7, 1]
    cs = plonk_circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = plonk_circuits.halo2lib_witness(cs, k, instances, lookup_bits=4, groups=40, num_gate_advice=3, num_lookup_advice=2)
    proofs = []
    for E in (plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree()), OracleEngine(k, cs.degree())):
        pk = plonk.keygen(E, cs, k, fixed, copies)
        rng = plonk.DeviceBulkRng(SeededRng(31), 0xc0ffee)
        proofs.append(plonk.create_proof(E, pk, [instances], adv, rng, EvmTranscriptWrite(pk.vk_digest)))
    assert proofs[0] == proofs[1]
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    assert plonk_verifier.verify(cs, k, pk.vk_digest, pk.fixed_commitments, pk.sigma_commitments, [instances], proofs[0], tau)
    other = plonk.create_proof(E, pk, [instances], adv, plonk.DeviceBulkRng(SeededRng(31), 0xc0ffef), EvmTranscriptWrite(pk.vk_digest))
    assert other != proofs[0]                                   # the seed matters


def _fixture_paths():
    import glob
    import os
    return sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "aggregation_k*_proof.json")))


@pytest.mark.parametrize("path", _fixture_paths(), ids=lambda p: p.split("_")[-2])
def test_k23_proof_equals_the_contract_accepted_fixture(be, orc, kats, path):
    """K = 23 / K = 24: the device regenerates, byte for byte, the proofs in tests/golden/aggregation_k2{3,4}_proof.json -- the
    ones the reference's sync_step / committee_update verifier contracts accepted when replayed by tests/yul_harness.py
    (tools/make_k23_fixture.py). The K = 24 proof needs most of an 80 GB device, so the workspaces and twiddle tables the
    other tests grew in the session's context are released first."""
    be.release_workspace()
    import json
    import os
    import time
    from spectre_b200 import plonk
    from spectre_b200.halo2 import ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from spectre_b200 import circuits as plonk_circuits
    from tests.plonk_oracle_engine import SeededRng
    with open(path) as f:
        fx = json.load(f)
    k = fx["k"]
    instances = [int(v, 16) for v in fx["instances"]]
    cs = plonk_circuits.aggregation_shape()
    fixed, adv, copies = plonk_circuits.aggregation_witness(cs, k, instances, fx["lookup_bits"], fx["groups"], seed=fx["seed"])
    params = ParamsKZG.setup(be, k, orc.srs_tau()).precompute()
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    t0 = time.perf_counter()
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=int(fx["vk_digest"]))
    t1 = time.perf_counter()
    timings = {}
    proof = plonk.create_proof(E, pk, [instances], [adv], SeededRng(fx["seed"]), EvmTranscriptWrite(pk.vk_digest), timings)
    t2 = time.perf_counter()
    print("K=%d keygen %.2fs create_proof %.2fs %s" % (k, t1 - t0, t2 - t1, {a: round(b, 3) for a, b in timings.items()}))
    assert [[hex(x), hex(y)] for x, y in pk.fixed_commitments + pk.sigma_commitments] == fx["vk_points"]
    kat = "range_table_commit_k%d_bits%d" % (k, fx["lookup_bits"])
    assert pk.fixed_commitments[1] == tuple(int(v, 16) for v in kats[kat]["xy"])                                # the contract's own VK constant
    assert proof.hex() == fx["proof"]
    del E, pk, params
    import torch
    torch.cuda.empty_cache()


@pytest.mark.parametrize("ids", device_lists())
def test_proof_with_msm_sharded_over_several_devices(orc, monkeypatch, ids):
    """One context driving several GPUs: every commitment of create_proof is an MSM sharded by point range (scalar ranges
    peer-copied over NVLink), the quotient kernels run on row ranges and the NTTs on whole polynomials spread over the
    devices (all through peer access to the first device's buffers; thresholds lowered so that this small circuit is
    actually sharded); the proof bytes do not change."""
    monkeypatch.setenv("SPB_SHARD_MIN_ROWS", "256")
    monkeypatch.setenv("SPB_SHARD_MIN_LOGN", "8")
    from spectre_b200 import circuits, halo2, plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import OracleEngine, SeededRng
    k, instances = 12, [3, 1, 4]
    cs = circuits.halo2lib_shape(4, 1)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=5, groups=200, num_gate_advice=4, num_lookup_advice=1)
    be2 = halo2.Backend(ids)
    try:
        proofs = []
        for E in (plonk.DeviceEngine(be2, halo2.ParamsKZG.setup(be2, k, orc.srs_tau()).precompute(), k, cs.degree()), OracleEngine(k, cs.degree())):
            pk = plonk.keygen(E, cs, k, fixed, copies)
            proofs.append(plonk.create_proof(E, pk, [instances], adv, SeededRng(5), EvmTranscriptWrite(pk.vk_digest)))
        assert proofs[0] == proofs[1]
    finally:
        be2.close()


@pytest.mark.parametrize("ids", device_lists())
@pytest.mark.parametrize("k", [10, 13])
def test_grand_products_sharded_by_row_range_over_the_devices(orc, monkeypatch, k, ids):
    """SURVEY.md 8e "grand product": on a context over several devices the permutation and lookup product columns are built per
    row range (terms, batch inversion and local products in each device's HBM, inputs read over NVLink), the range totals are the
    one exchange, and the seeded scans write their slices of z into the first device's buffer: the columns -- blinding tail and
    the chained last_z included -- equal the oracle's, i.e. the one-device scan, bit for bit."""
    import torch
    monkeypatch.setenv("SPB_SHARD_MIN_ROWS", "256")
    from spectre_b200 import halo2
    be2 = halo2.Backend(ids)
    try:
        n, n_cols, chunk, n_blinds = 1 << k, 5, 2, 5
        values = [orc.fr_random_chacha(n, 100 + c) for c in range(n_cols)]
        sigma = [orc.fr_random_chacha(n, 200 + c) for c in range(n_cols)]
        values[0][3] = 0; sigma[0][5] = 0
        beta, gamma = orc.fr_random_chacha(2, 300 + k)
        dv, ds = [_dev(torch, a) for a in values], [_dev(torch, a) for a in sigma]
        dz = torch.empty((n, 4), dtype=torch.int64, device="cuda:0")
        last_o = last_g = orc.fr([1])[0]
        for s_, lo in enumerate(range(0, n_cols, chunk)):
            hi = min(lo + chunk, n_cols)
            blinds = orc.fr_random_chacha(n_blinds, 400 + s_).reshape(-1, 4)
            z_want, last_o = orc.permutation_product(k, values[lo:hi], sigma[lo:hi], lo, beta, gamma, blinds, last_o)
            last_g = be2.permutation_product_dev(k, [t.data_ptr() for t in dv[lo:hi]], [t.data_ptr() for t in ds[lo:hi]], lo, beta, gamma, blinds, last_g, dz.data_ptr())
            assert np.array_equal(_host(dz), z_want)
            assert np.array_equal(last_g, last_o.reshape(4))
        arrs = [orc.fr_random_chacha(n, 500 + i) for i in range(4)]
        arrs[3][9] = orc.fr([-orc.fr_ints(gamma.reshape(1, 4))[0]])[0]
        blinds = orc.fr_random_chacha(n_blinds, 602).reshape(-1, 4)
        d = [_dev(torch, a) for a in arrs]
        be2.lookup_product_dev(n, *[t.data_ptr() for t in d], beta, gamma, blinds, dz.data_ptr())
        assert np.array_equal(_host(dz), orc.lookup_product(*arrs, beta, gamma, blinds))
    finally:
        torch.cuda.synchronize()
        be2.close()


def test_lookup_violation_is_reported_like_upstream(be, orc):
    """an advice value outside the table: permute_expression_pair fails (upstream: Error::ConstraintSystemFailure) and
    create_proof raises instead of producing a proof"""
    from spectre_b200 import circuits, plonk
    from spectre_b200.halo2 import BackendError, ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    k, instances = 7, [1]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, lookup_bits=3, groups=10)
    adv[4] = plonk.fr_mont(99)                                  # a looked-up cell (q_lookup = 1 on row 4) outside [0, 8)
    E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    with pytest.raises(BackendError):
        plonk.create_proof(E, pk, [instances], [adv], SeededRng(2), EvmTranscriptWrite(pk.vk_digest))


def test_proving_key_file_streams_between_disk_and_hbm(be, orc, tmp_path):
    """*.pkey through spb_write_file_dev / spb_read_file_dev (double-buffered pinned staging): the file the device writes is
    byte-identical to the one the CPU oracle engine writes for the same key, and the key read back into HBM proves to the
    same bytes. Also ParamsKZG::write / ::read through the same streamer."""
    from spectre_b200 import circuits, plonk
    from spectre_b200.halo2 import ParamsKZG
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import OracleEngine, SeededRng
    k, instances = 9, [3, 1, 4]
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=4, groups=40, num_gate_advice=3, num_lookup_advice=2)
    params = ParamsKZG.setup(be, k, orc.srs_tau())
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    dev_path, cpu_path = str(tmp_path / "dev.pkey"), str(tmp_path / "cpu.pkey")
    plonk.write_pk(E, pk, dev_path)
    Ec = OracleEngine(k, cs.degree())
    plonk.write_pk(Ec, plonk.keygen(Ec, cs, k, fixed, copies), cpu_path)
    with open(dev_path, "rb") as f1, open(cpu_path, "rb") as f2:
        assert f1.read() == f2.read()
    pk2 = plonk.read_pk(E, cs, cpu_path)
    proofs = [plonk.create_proof(E, key, [instances], adv, SeededRng(4), EvmTranscriptWrite(key.vk_digest)) for key in (pk, pk2)]
    assert proofs[0] == proofs[1]
    # params file round trip through the same streamer
    ppath = str(tmp_path / ("kzg_bn254_%d.srs" % k))
    params.write(ppath)
    back = ParamsKZG.read(be, ppath)
    assert np.array_equal(back.get_g(), params.get_g()) and np.array_equal(back.get_g(basis=1), params.get_g(basis=1))
