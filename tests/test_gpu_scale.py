"""Kernel paths that only run at production sizes, compared bit for bit with the CPU oracle (oracle/halo2_oracle.c) or
Python integers. The oracle is the reference here, never the thing under test.

* Quotient kernels past one grid of rows. graph_evaluate_kernel grid-strides 2 x SMs x 256 thread slots over the rows and
  keeps each slot's intermediates at scratch[i * nslots + slot]; permutation_constraints_kernel builds extended_omega^row
  from one power per 256-row block. Below E = 2^17 no slot takes a second row and only the first blocks run.
* spb_eval_polynomial_many_dev / spb_eval_polynomial_dev across the sizes where their thread count T changes.
* The device-resident EvaluationDomain entry points create_proof calls, with guard rows after every output.
* The two-level twiddle tables, which an NTT at k >= 12 only uses once the cached full tables fill their per-device budget.
* Sync-step-shaped proofs (halo2lib_shape) whose extended domains take several grids.
"""
import functools
import random
import time

import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be  # noqa: F401
from tests.quotient_common import random_program

pytestmark = pytest.mark.gpu

R = pyref.R_MOD
GUARD = 64                                                                  # sentinel rows after every output buffer
SENTINEL = int(np.array([0xA5A5A5A5A5A5A5A5], dtype=np.uint64).view(np.int64)[0])


@pytest.fixture(scope="module", autouse=True)
def _free_module_buffers():
    yield
    _pool.cache_clear()
    import torch
    torch.cuda.empty_cache()


def _residues(rows, seed):
    """(rows, 4) Montgomery limbs of random field elements: uniform low limbs, top limb below r's, so every value is < r"""
    g = np.random.default_rng(seed)
    a = np.frombuffer(g.bytes(rows * 32), dtype=np.uint64).reshape(rows, 4).copy()
    a[:, 3] = g.integers(0, R >> 192, size=rows, dtype=np.uint64)
    return a


def _up(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def _down(t):
    return t.cpu().numpy().view(np.uint64)


def _guarded(torch, rows, fill=None):
    """rows + GUARD rows of SENTINEL on the device; `fill` (host rows) goes into the first rows"""
    t = torch.full((rows + GUARD, 4), SENTINEL, dtype=torch.int64, device="cuda")
    if fill is not None:
        t[:fill.shape[0]] = _up(torch, fill)
    return t


def _check_guarded(t, rows, want, what):
    got = _down(t)
    assert np.array_equal(got[:rows], want), what
    assert (got[rows:].view(np.int64) == SENTINEL).all(), "%s wrote past its %d rows" % (what, rows)


# ---- 1. quotient kernels past one grid -------------------------------------------------------------------------------
QUOTIENT_SIZES = [1 << 17, 1 << 19]     # E = 2^17: 1-2 rows per thread slot on 132 SMs; 2^19: about 8
ROT_SCALE = 4
POOL = 60


@functools.lru_cache(maxsize=2)
def _pool(E):
    """POOL distinct random columns of E rows, on the host and on the device"""
    import torch
    host = [_residues(E, (E << 8) + i) for i in range(POOL)]
    return host, [_up(torch, a) for a in host]


def _graph_case(orc, name):
    """-> (program words, #calculations, constants, rotations, (#fixed, #advice, #instance), challenges)"""
    from spectre_b200 import circuits
    if name == "random150":
        bf = circuits.halo2lib_shape().blinding_factors()
        rotations = np.array([0, 1, -1, 2, 3, -(bf + 1)], dtype=np.int32)
        constants = _residues(5, 5); constants[0] = 0; constants[1] = orc.fr([1])[0]
        prog = random_program(random.Random(150), 150, len(constants), len(rotations), 3, 4, 1, 2)
        return prog, 150, constants, rotations, (3, 4, 1), _residues(2, 6)
    cs = circuits.aggregation_shape() if name == "aggregation_gate" else circuits.halo2lib_shape()
    if name == "spread_lookup":
        li = len(cs.lookups) - 1
        assert len(cs.lookups[li][0]) == 2                                 # the two-column lookup compressed with theta
        p = cs.lookup_value_program(li)
    else:
        p = cs.gates_program()
    # the gates query rotations 0..3; rotations 1 and 2 become -1 and -(bf+1) so that row indices wrap at both ends
    bf = cs.blinding_factors()
    rotations = np.array([{1: -1, 2: -(bf + 1)}.get(int(r), int(r)) for r in p["rotations"]], dtype=np.int32)
    return p["prog"], p["ncalc"], p["constants"], rotations, (cs.num_fixed, cs.num_advice, cs.num_instance), np.zeros((1, 4), np.uint64)


@pytest.mark.parametrize("E", QUOTIENT_SIZES)
@pytest.mark.parametrize("name", ["halo2lib_gates", "spread_lookup", "aggregation_gate", "random150"])
def test_graph_evaluate_past_one_grid(be, orc, name, E):
    import torch
    prog, ncalc, constants, rotations, (nf, na, ni), challenges = _graph_case(orc, name)
    host, dev = _pool(E)
    cols = lambda xs, lo, cnt: xs[lo:lo + cnt]
    bgty = _residues(4, 7)
    want = orc.graph_evaluate(prog, ncalc, ncalc, constants, rotations, cols(host, 0, nf), cols(host, nf, na), cols(host, nf + na, ni), challenges, bgty,
                              host[POOL - 1], ROT_SCALE)
    dv = dev[POOL - 1].clone()
    ptrs = lambda ts: [t.data_ptr() for t in ts]
    torch.cuda.synchronize()
    be.graph_evaluate_dev(prog, ncalc, ncalc, constants, rotations, ptrs(cols(dev, 0, nf)), ptrs(cols(dev, nf, na)), ptrs(cols(dev, nf + na, ni)),
                          challenges, bgty[0], bgty[1], bgty[2], bgty[3], dv.data_ptr(), E, ROT_SCALE)
    assert np.array_equal(_down(dv), want)


@pytest.mark.parametrize("E", QUOTIENT_SIZES)
def test_permutation_constraints_past_one_grid(be, orc, E):
    """the sync-step shape's permutation: 21 columns in 11 sets of 2, last rotation -(bf+1), extended_omega of Domain(4, k)"""
    import torch
    from spectre_b200 import circuits
    cs = circuits.halo2lib_shape()
    n_cols, chunk = len(cs.permutation), cs.chunk_len()
    n_sets = -(-n_cols // chunk)
    assert (n_cols, chunk, n_sets) == (21, 2, 11)
    last_rotation = -(cs.blinding_factors() + 1)
    od = orc.Domain(4, E.bit_length() - 3)
    assert od.extended_k == E.bit_length() - 1
    host, dev = _pool(E)
    z, cv, sg, rest = slice(0, 11), slice(11, 32), slice(32, 53), (53, 54, 55)
    beta, gamma, y = _residues(3, 8)
    want = orc.permutation_constraints(host[POOL - 1], ROT_SCALE, last_rotation, chunk, host[z], host[cv], host[sg], *[host[i] for i in rest], beta, gamma, y,
                                       od.extended_omega)
    dv = dev[POOL - 1].clone()
    ptrs = lambda ts: [t.data_ptr() for t in ts]
    torch.cuda.synchronize()
    be.permutation_constraints_dev(dv.data_ptr(), E, ROT_SCALE, last_rotation, chunk, ptrs(dev[z]), ptrs(dev[cv]), ptrs(dev[sg]), *[dev[i].data_ptr() for i in rest],
                                   beta, gamma, y, od.extended_omega)
    assert np.array_equal(_down(dv), want)


@pytest.mark.parametrize("E", QUOTIENT_SIZES)
def test_lookup_constraints_past_one_grid(be, orc, E):
    import torch
    host, dev = _pool(E)
    beta, gamma, y = _residues(3, 9)
    want = orc.lookup_constraints(host[POOL - 1], ROT_SCALE, *host[:7], beta, gamma, y)
    dv = dev[POOL - 1].clone()
    torch.cuda.synchronize()
    be.lookup_constraints_dev(dv.data_ptr(), E, ROT_SCALE, *[t.data_ptr() for t in dev[:7]], beta, gamma, y)
    assert np.array_equal(_down(dv), want)


# ---- 2. polynomial evaluation across thread-count boundaries ---------------------------------------------------------
# eval_many: T = 256 .. 16384 (T * 64 >= n), Horner chains longer than 64 above n = 2^20; eval single: T up to 65536 (T * 16 >= n)
EVAL_SIZES = [1, 2, 255, 256, 257, 16384, 16385, 1 << 19, (1 << 19) + 1, (1 << 20) + 1, 1 << 22]
N_POLYS = 4


def _eval_queries(count, k):
    """`count` (polynomial index, point) queries in the order create_proof issues them: one polynomial pointer opened at x, omega x,
    omega^-1 x and omega^-(bf+1) x (bf = 6 in the sync-step shape), then the next; every third group of four opens at the
    points 0, 1, omega and omega^5 instead. Two distinct x alternate, so no two neighbouring groups share points."""
    w = pyref.omega(k)
    rots = [1, w, pow(w, -1, R), pow(w, -7, R)]
    xs = [pow(0x5eed, 11, R), pow(0xfeed, 13, R)]
    specials = [0, 1, w, pow(w, 5, R)]
    out = []
    for i in range(count):
        b, pos = divmod(i, 4)
        kind = b % 3
        out.append((b % N_POLYS, specials[pos] if kind == 2 else xs[kind] * rots[pos] % R))
    return out


def _eval_many_and_reference(be, orc, polys, dpolys, n, queries, ref):
    got = be.eval_polynomial_many_dev([dpolys[i].data_ptr() for i, _ in queries], n, orc.fr([pt for _, pt in queries]))
    for key in queries:
        if key not in ref:
            ref[key] = orc.eval_polynomial(polys[key[0]], orc.fr([key[1]])[0])
    return got, np.stack([ref[key] for key in queries])


@pytest.mark.parametrize("n", EVAL_SIZES)
def test_eval_polynomial_many_across_thread_counts(be, orc, n):
    import torch
    polys = [_residues(n, (n << 4) + i) for i in range(N_POLYS)]
    dpolys = [_up(torch, p) for p in polys]
    torch.cuda.synchronize()
    queries, ref = _eval_queries(153, max(1, (n - 1).bit_length())), {}
    for count in (1, 3, 153):
        got, want = _eval_many_and_reference(be, orc, polys, dpolys, n, queries[:count], ref)
        assert np.array_equal(got, want), "count %d" % count


@pytest.mark.parametrize("n", [(1 << 20) + 1, 1 << 22])
def test_eval_polynomial_dev_at_the_thread_cap(be, orc, n):
    import torch
    poly = _residues(n, n)
    dp = _up(torch, poly)
    torch.cuda.synchronize()
    w = pyref.omega(max(1, (n - 1).bit_length()))
    for pt in (pow(0x5eed, 11, R), w, pow(w, -7, R), 0, 1):
        x = orc.fr([pt])[0]
        assert np.array_equal(be.eval_polynomial_dev(dp.data_ptr(), n, x), orc.eval_polynomial(poly, x)), hex(pt)


def test_eval_polynomial_many_query_limits(be, orc):
    """65535 queries (the grid's y limit) are accepted and right; 65536 queries and n = 0 are argument errors"""
    import torch
    from spectre_b200.halo2 import BackendError
    n = 257
    polys = [_residues(n, 77 + i) for i in range(N_POLYS)]
    dpolys = [_up(torch, p) for p in polys]
    torch.cuda.synchronize()
    got, want = _eval_many_and_reference(be, orc, polys, dpolys, n, _eval_queries(65535, 9), {})
    assert np.array_equal(got, want)
    with pytest.raises(BackendError):
        be.eval_polynomial_many_dev([dpolys[0].data_ptr()] * 65536, n, np.zeros((65536, 4), np.uint64))
    with pytest.raises(BackendError):
        be.eval_polynomial_many_dev([dpolys[0].data_ptr()], 0, np.zeros((1, 4), np.uint64))


# ---- 3. the device-resident domain operations ------------------------------------------------------------------------
# (4, k): the sync-step shape, extended_to_coeff keeps 3/4 of the rows; (5, 16): the aggregation shape, it keeps all of them.
# (4, 21) is E = 2^23: three passes of 2^11-element tiles, one CTA per tile.
DOMAIN_CASES = [(4, 12), (4, 17), (4, 20), (4, 21), (5, 16)]


def _npass(k):
    """passes of a 2^k NTT: digits of at most 11 bits (ntt_make_plan with kMaxDigitBits in csrc/ntt.cu)"""
    return 1 if k <= 11 else -(-k // 11)


class _TwoLevelTables:
    """Expected kernel launches of NTTs made while the full-table budget is spent: npass(k) per transform, plus the two
    power-table launches of get_tables the first time a (k, omega) pair is seen -- and no third, full-table, launch."""

    def __init__(self):
        self.seen = set()

    def expect(self, k, omega, count=1):
        key = (k, np.ascontiguousarray(omega, dtype=np.uint64).tobytes())
        new = key not in self.seen
        self.seen.add(key)
        return count * _npass(k) + (2 if new else 0)


def _launches(be, tables, k, omega, count, fn):
    before = be.kernel_launches
    fn()
    if tables is not None:
        assert be.kernel_launches - before == tables.expect(k, omega, count), "2^%d transform: unexpected table launches" % k


def _domain_ops(be, orc, j, k, seed, tables=None):
    """lagrange_to_coeff_batch_dev, coeff_to_extended_dev, coeff_to_extended_batch_dev, extended_to_coeff_dev and
    divide_by_vanishing_poly_dev against orc.Domain. Batches of 1, 2 and 5 distinct buffers: member i holds the first member's
    input times a random scalar, so (the transforms being linear) its reference is the first reference times that scalar."""
    import torch
    from spectre_b200.halo2 import EvaluationDomain
    d, od = EvaluationDomain(be, j, k), orc.Domain(j, k)
    n, ek = 1 << k, d.extended_k
    E, kept = 1 << ek, (j - 1) << k
    assert ek == od.extended_k and kept <= E
    scales = _residues(4, seed + 1)
    members = lambda a: [a] + [orc.vec_scale(a, s) for s in scales]
    ptrs = lambda ts: [t.data_ptr() for t in ts]

    lag = _residues(n, seed + 2)
    ins, wants = members(lag), members(od.lagrange_to_coeff(lag))
    for count in (1, 2, 5):
        bufs = [_guarded(torch, n, a) for a in ins[:count]]
        torch.cuda.synchronize()
        _launches(be, tables, k, d.omega_inv, count, lambda: d.lagrange_to_coeff_batch_dev(ptrs(bufs)))
        for i, b in enumerate(bufs):
            _check_guarded(b, n, wants[i], "lagrange_to_coeff_batch_dev(%d, %d) member %d of %d" % (j, k, i, count))
    del bufs

    # coefficients are the first 2^k rows of an E-row tensor whose tail holds random non-zero residues: the transform must
    # zero-pad, not read them
    coeff, tail = _residues(n, seed + 3), _residues(E - n, seed + 4)
    assert not (tail == 0).all(axis=1).any()
    dtail = _up(torch, tail)
    ins, wants = members(coeff), members(od.coeff_to_extended(coeff))
    src = torch.cat([_up(torch, coeff), dtail])
    out = _guarded(torch, E)
    torch.cuda.synchronize()
    _launches(be, tables, ek, d.extended_omega, 1, lambda: d.coeff_to_extended_dev(src.data_ptr(), out.data_ptr()))
    _check_guarded(out, E, wants[0], "coeff_to_extended_dev(%d, %d)" % (j, k))
    assert np.array_equal(_down(src[n:]), tail)
    del src, out
    for count in (1, 2, 5):
        srcs = [torch.cat([_up(torch, a), dtail]) for a in ins[:count]]
        outs = [_guarded(torch, E) for _ in range(count)]
        torch.cuda.synchronize()
        _launches(be, tables, ek, d.extended_omega, count, lambda: d.coeff_to_extended_batch_dev(ptrs(srcs), ptrs(outs)))
        for i, o in enumerate(outs):
            _check_guarded(o, E, wants[i], "coeff_to_extended_batch_dev(%d, %d) member %d of %d" % (j, k, i, count))
        del srcs, outs
    del dtail

    ext = _residues(E, seed + 5)
    src, out = _up(torch, ext), _guarded(torch, kept)
    torch.cuda.synchronize()
    _launches(be, tables, ek, d.extended_omega_inv, 1, lambda: d.extended_to_coeff_dev(src.data_ptr(), out.data_ptr()))
    _check_guarded(out, kept, od.extended_to_coeff(ext), "extended_to_coeff_dev(%d, %d)" % (j, k))
    del src, out

    buf = _guarded(torch, E, ext)
    torch.cuda.synchronize()
    before = be.kernel_launches
    d.divide_by_vanishing_poly_dev(buf.data_ptr())
    assert be.kernel_launches - before == 1
    _check_guarded(buf, E, od.divide_by_vanishing_poly(ext), "divide_by_vanishing_poly_dev(%d, %d)" % (j, k))


@pytest.mark.parametrize("j,k", DOMAIN_CASES)
def test_device_domain_operations(be, orc, j, k):
    _domain_ops(be, orc, j, k, seed=1000 * j + k)


# ---- 4. two-level twiddle tables, forced and observed ----------------------------------------------------------------
def test_two_level_twiddle_tables(be, orc):
    """Six k = 25 transforms under distinct primitive roots cache 6 x 1 GiB of full omega^i tables, the whole per-device budget
    (kFullTableBudget, 6 GiB). Every table made after that is two-level (ntt_omega_pow multiplies a high and a low entry):
    best_fft_dev at k = 12..23 and the (4, 20) domain operations must still match the oracle, and the launch counts show which
    branch get_tables took. The same transform with a full table (after a release) gives the same bits."""
    import torch
    be.release_workspace()
    try:
        k_fill = 25
        n = 1 << k_fill
        w = pyref.omega(k_fill)
        src = _up(torch, _residues(n, 2525))
        buf = torch.empty_like(src)
        for i in range(6):
            wi = orc.fr([pow(w, 2 * i + 1, R)])[0]
            buf.copy_(src)
            torch.cuda.synchronize()
            before = be.kernel_launches
            be.best_fft_dev(buf.data_ptr(), wi, k_fill)
            assert be.kernel_launches - before == 3 + _npass(k_fill), "k = 25 transform %d did not get a full table" % i
            assert np.array_equal(_down(buf[1:2])[0], be.eval_polynomial_dev(src.data_ptr(), n, wi)), "X[1] != p(omega') for root %d" % i
        del src, buf
        torch.cuda.empty_cache()

        tables, two_level = _TwoLevelTables(), {}
        for k in (12, 18, 20, 21, 22, 23):
            a, wk = _residues(1 << k, 600 + k), orc.fr([pyref.omega(k)])[0]
            da = _up(torch, a)
            torch.cuda.synchronize()
            before = be.kernel_launches
            be.best_fft_dev(da.data_ptr(), wk, k)
            assert be.kernel_launches - before == tables.expect(k, wk) == 2 + _npass(k), "2^%d: not a two-level table" % k
            two_level[k] = (a, _down(da))
            assert np.array_equal(two_level[k][1], orc.best_fft(a, wk, k)), "2^%d" % k
            del da
        _domain_ops(be, orc, 4, 20, seed=4020, tables=tables)

        be.release_workspace()
        k = 23
        a, want = two_level[k]
        da = _up(torch, a)
        torch.cuda.synchronize()
        before = be.kernel_launches
        be.best_fft_dev(da.data_ptr(), orc.fr([pyref.omega(k)])[0], k)
        assert be.kernel_launches - before == 3 + _npass(k), "2^23 after a release: expected a full table"
        assert np.array_equal(_down(da), want)
    finally:
        be.release_workspace()
        torch.cuda.empty_cache()


# ---- 5. sync-step-shaped proofs beyond one grid ----------------------------------------------------------------------
_device_proofs = {}     # k -> (vk digest, fixed commitments, sigma commitments, proof): the slow oracle comparison reuses it


def _sync_step_case(k):
    """halo2lib_shape() with the witness recipe of bench.py's sync-step case"""
    from spectre_b200 import circuits
    cs = circuits.halo2lib_shape()
    inst = list(range(1, 15))
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, min(16, k - 2), 500, seed=1)
    return cs, inst, fixed, adv, copies


def _prove(E, cs, k, inst, fixed, adv, copies):
    from spectre_b200 import plonk
    from spectre_b200.transcript import EvmTranscriptWrite
    from tests.plonk_oracle_engine import SeededRng
    pk = plonk.keygen(E, cs, k, fixed, copies)
    proof = plonk.create_proof(E, pk, [inst], adv, SeededRng(20 + k), EvmTranscriptWrite(pk.vk_digest))
    return (pk.vk_digest, pk.fixed_commitments, pk.sigma_commitments, proof)


def _device_proof(be, orc, k, case):
    if k not in _device_proofs:
        import torch
        from spectre_b200 import plonk
        from spectre_b200.halo2 import ParamsKZG
        cs = case[0]
        E = plonk.DeviceEngine(be, ParamsKZG.setup(be, k, orc.srs_tau()), k, cs.degree())
        _device_proofs[k] = _prove(E, k=k, cs=cs, inst=case[1], fixed=case[2], adv=case[3], copies=case[4])
        del E
        torch.cuda.empty_cache()
    return _device_proofs[k]


def _oracle_proof(k, case):
    from tests.plonk_oracle_engine import OracleEngine
    t0 = time.perf_counter()
    out = _prove(OracleEngine(k, case[0].degree()), case[0], k, *case[1:])
    print("oracle engine keygen + create_proof, halo2lib shape k = %d: %.1f s on the host" % (k, time.perf_counter() - t0))
    return out


def _verifies(orc, cs, k, inst, vk):
    from tests import plonk_verifier
    digest, fixed_c, sigma_c, proof = vk
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    return plonk_verifier.verify(cs, k, digest, fixed_c, sigma_c, [inst], proof, tau)


def test_sync_step_proof_k16_matches_the_oracle_and_verifies(be, orc):
    """k = 16: E = 2^18 extended rows, four grids of graph_evaluate thread slots"""
    k = 16
    case = _sync_step_case(k)
    dev = _device_proof(be, orc, k, case)
    assert dev == _oracle_proof(k, case)
    assert _verifies(orc, case[0], k, case[1], dev)


def test_sync_step_proof_k20_verifies(be, orc):
    """k = 20, the size bench.py times: the independent verifier accepts the device proof"""
    k = 20
    case = _sync_step_case(k)
    assert _verifies(orc, case[0], k, case[1], _device_proof(be, orc, k, case))


@pytest.mark.slow
def test_sync_step_proof_k20_matches_the_oracle(be, orc):
    k = 20
    case = _sync_step_case(k)
    assert _device_proof(be, orc, k, case) == _oracle_proof(k, case)
