"""Device-resident `keygen_pk` / `create_proof`: the host-side mirror of halo2's prover driver over the C ABI
(SURVEY.md 8f row 1 "device-resident proving pipeline", rows a6-a9 of 8a).

  [UPSTREAM] halo2_proofs/src/plonk/keygen.rs  keygen_pk            -> keygen()
  [UPSTREAM] halo2_proofs/src/plonk/prover.rs  create_proof          -> create_proof()
  [UPSTREAM] .../poly/kzg/multiopen/shplonk.rs construct_intermediate_sets -> rotation_sets()

reached in the reference from lightclient-circuits/src/util/circuit.rs:131,158,211 through snark_verifier_sdk.
What lives here is what the Rust shim of INTEGRATION.md keeps on the host: the order of the protocol, the transcript,
the RNG draws, the (tiny) rotation-set bookkeeping. Every polynomial lives in HBM from the moment its column is
uploaded; per stage only challenges, blinding values, 32-byte evaluations and 96-byte commitments cross the ABI.

The driver is written against a small engine interface (`DeviceEngine` below binds it to libspectre_b200.so); the
parity tests bind the same driver to the CPU oracle and require byte-identical proofs, and an independent verifier
(tests/plonk_verifier.py, and the reference's own verifier contract replayed in tests/yul_harness.py) accepts them.

A circuit is described by a `ConstraintSystem` of expression trees -- the information `pk.get_vk().cs()` holds
upstream. Expressions are nested tuples built with Const / Fixed / Advice / Instance / Neg / Sum / Prod / Scaled.
"""
import secrets
from collections import namedtuple

import numpy as np

from . import halo2

R_MOD = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
P_MOD = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
_MONT = (1 << 256) % R_MOD
_MONT_INV = pow(_MONT, -1, R_MOD)
ROOT_OF_UNITY = pow(7, (R_MOD - 1) >> 28, R_MOD)
DELTA = pow(7, 1 << 28, R_MOD)
ZETA = pow(pow(7, (R_MOD - 1) // 3, R_MOD), 2, R_MOD)       # the extended coset's shift (EvaluationDomain g_coset)

# flat GraphEvaluator encoding (include/spectre_b200.h)
ADD, SUB, MUL, SQUARE, DOUBLE, NEGATE, HORNER, STORE = range(8)
K_CONST, K_INTER, K_FIXED, K_ADVICE, K_INSTANCE, K_CHALLENGE, K_BETA, K_GAMMA, K_THETA, K_Y, K_PREV = range(11)


def fr_mont(v):
    """Python int -> (4,) uint64 Montgomery limbs (the in-memory form of halo2curves' Fr)."""
    m = (v % R_MOD) * _MONT % R_MOD
    return np.array([(m >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)


def fr_int(a):
    a = np.asarray(a, dtype=np.uint64).reshape(4)
    return (int(a[0]) | int(a[1]) << 64 | int(a[2]) << 128 | int(a[3]) << 192) * _MONT_INV % R_MOD


def fr_mont_rows(vals):
    return np.stack([fr_mont(v) for v in vals]) if len(vals) else np.zeros((0, 4), dtype=np.uint64)


def omega_of(k):
    return pow(ROOT_OF_UNITY, 1 << (28 - k), R_MOD)


# ---- expressions ------------------------------------------------------------------------------------------------
def Const(v): return ("const", v % R_MOD)
def Fixed(c, rot=0): return ("fixed", c, rot)
def Advice(c, rot=0): return ("advice", c, rot)
def Instance(c, rot=0): return ("instance", c, rot)
def Neg(e): return ("neg", e)
def Sum(a, b): return ("sum", a, b)
def Prod(a, b): return ("prod", a, b)
def Scaled(e, v): return ("scaled", e, v % R_MOD)


def degree(e):
    t = e[0]
    if t == "const": return 0
    if t in ("fixed", "advice", "instance"): return 1
    if t in ("neg", "scaled"): return degree(e[1])
    if t == "sum": return max(degree(e[1]), degree(e[2]))
    return degree(e[1]) + degree(e[2])


def queries(e, out):
    """column queries of an expression in first-seen order -> out: {kind: [(col, rot), ...]}"""
    t = e[0]
    if t in ("fixed", "advice", "instance"):
        q = (e[1], e[2])
        if q not in out[t]:
            out[t].append(q)
    elif t in ("neg", "scaled"):
        queries(e[1], out)
    elif t in ("sum", "prod"):
        queries(e[1], out); queries(e[2], out)


class Program:
    """Builder of one flat GraphEvaluator program."""

    def __init__(self):
        self.words, self.ncalc, self.constants, self.rotations = [], 0, [0, 1], []
        self.seen = {}   # (op, sources) -> intermediate: identical calculations are emitted once (GraphEvaluator::add_calculation)

    def _const(self, v):
        if v not in self.constants:
            self.constants.append(v)
        return (K_CONST, self.constants.index(v))

    def _rot(self, r):
        if r not in self.rotations:
            self.rotations.append(r)
        return self.rotations.index(r)

    def _emit(self, op, srcs, nparts=0):
        key = (op, nparts, tuple(srcs))
        if key in self.seen:
            return self.seen[key]
        self.seen[key] = (K_INTER, self.ncalc)
        self.words += [op | (nparts << 8), self.ncalc]
        for s in srcs:
            self.words += [s[0], s[1]]
        self.ncalc += 1
        return (K_INTER, self.ncalc - 1)

    def src(self, e):
        t = e[0]
        if t == "const": return self._const(e[1])
        if t == "fixed": return (K_FIXED, e[1] | (self._rot(e[2]) << 16))
        if t == "advice": return (K_ADVICE, e[1] | (self._rot(e[2]) << 16))
        if t == "instance": return (K_INSTANCE, e[1] | (self._rot(e[2]) << 16))
        if t == "neg": return self._emit(NEGATE, [self.src(e[1])])
        if t == "sum": return self._emit(ADD, [self.src(e[1]), self.src(e[2])])
        if t == "prod": return self._emit(MUL, [self.src(e[1]), self.src(e[2])])
        if t == "scaled": return self._emit(MUL, [self.src(e[1]), self._const(e[2])])
        raise ValueError("unknown expression node %r" % (t,))

    def horner(self, start, factor, exprs):
        parts = [self.src(e) for e in exprs]
        return self._emit(HORNER, [start, factor] + parts, nparts=len(parts))

    def finish(self):
        return dict(prog=np.array(self.words, dtype=np.uint32), ncalc=self.ncalc, constants=fr_mont_rows(self.constants),
                    rotations=np.array(self.rotations or [0], dtype=np.int32))


class ConstraintSystem:
    """What halo2's ConstraintSystem records at configure time, for the parts create_proof reads."""

    def __init__(self, num_fixed, num_advice, num_instance, gates, lookups, permutation, fixed_queries=None, advice_queries=None, minimum_degree=None):
        self.num_fixed, self.num_advice, self.num_instance = num_fixed, num_advice, num_instance
        self.minimum_degree = minimum_degree                               # ConstraintSystem::set_minimum_degree
        self.gates, self.lookups, self.permutation = list(gates), [(list(i), list(t)) for i, t in lookups], list(permutation)
        q = {"fixed": list(fixed_queries or []), "advice": list(advice_queries or []), "instance": []}
        for g in self.gates:
            queries(g, q)
        for ins, tbs in self.lookups:
            for e in ins + tbs:
                queries(e, q)
        for kind, col in self.permutation:         # enable_equality queries the column at Rotation::cur()
            if (col, 0) not in q[kind]:
                q[kind].append((col, 0))
        self.fixed_queries, self.advice_queries, self.instance_queries = q["fixed"], q["advice"], q["instance"]

    def degree(self):
        """ConstraintSystem::degree ([UPSTREAM] halo2_proofs/src/plonk/circuit.rs): the permutation argument's
        required_degree() = 3 always enters, equality columns or not; a lookup needs max(4, 2 + input_degree + table_degree)
        with both degrees floored at 1; then the gates; finally `minimum_degree` if the circuit set one."""
        d = 3                                                               # permutation::Argument::required_degree
        for ins, tbs in self.lookups:                                      # lookup::Argument::required_degree
            d = max(d, max(4, 2 + max([1] + [degree(e) for e in ins]) + max([1] + [degree(e) for e in tbs])))
        for g in self.gates:
            d = max(d, degree(g))
        return max(d, self.minimum_degree or 0)

    def blinding_factors(self):
        per_col = [sum(1 for c, _ in self.advice_queries if c == col) for col in range(self.num_advice)]
        return max(3, max(per_col or [1])) + 2

    def chunk_len(self):
        return self.degree() - 2

    # programs ---------------------------------------------------------------------------------------------------
    def gates_program(self):
        p = Program()
        p.horner((K_PREV, 0), (K_Y, 0), self.gates)
        return p.finish()

    def lookup_compress_program(self, exprs):
        p = Program()
        p.horner(p._const(0), (K_THETA, 0), exprs)
        return p.finish()

    def lookup_value_program(self, li):
        ins, tbs = self.lookups[li]
        p = Program()
        a = p.horner(p._const(0), (K_THETA, 0), ins)
        s = p.horner(p._const(0), (K_THETA, 0), tbs)
        p._emit(MUL, [p._emit(ADD, [a, (K_BETA, 0)]), p._emit(ADD, [s, (K_GAMMA, 0)])])
        return p.finish()


def uniform_residues(torch, rows, device, generator=None):
    """(rows, 4) int64 tensor of uniformly random Fr elements generated ON `device` (rejection sampling of 254-bit
    candidates against r; a uniform residue is a uniform field element in Montgomery form too). Used for the vanishing
    argument's random polynomial: at K = 23 that is 256 MiB that never has to be drawn on the host or cross PCIe.
    Candidates whose top limb equals r's top limb are rejected outright (probability 2^-62)."""
    r3 = R_MOD >> 192
    out, have = [], 0
    while have < rows:
        m = int((rows - have) * 1.4) + 64
        c = torch.randint(-(1 << 63), (1 << 63) - 1, (m, 4), dtype=torch.int64, device=device, generator=generator)
        c[:, 3] = torch.randint(0, 1 << 62, (m,), dtype=torch.int64, device=device, generator=generator)
        keep = c[c[:, 3] < r3]
        out.append(keep); have += keep.shape[0]
    return torch.cat(out)[:rows].contiguous()


class DeviceBulkRng:
    """The `rng` argument of create_proof with its one bulk draw kept in HBM: blinding rows come from `host_rng(count)` (a
    few rows per column), the vanishing argument's 2^k-coefficient random polynomial from the engine's ChaCha20 stream of
    `seed` (Engine.random_chacha -> spb_fr_random_chacha_dev: `Fr::random(ChaCha20Rng::from_seed(seed))` draws 0..2^k-1), so
    it is never drawn on the host and never crosses PCIe. Upstream passes OsRng here
    (lightclient-circuits/src/util/circuit.rs:158,211); any CSPRNG stream is as good."""

    def __init__(self, host_rng, seed):
        self.host_rng = host_rng
        self.seed = seed.to_bytes(32, "little") if isinstance(seed, int) else bytes(seed)

    def __call__(self, count):
        return self.host_rng(count)

    def device_rows(self, E, count):
        return E.random_chacha(self.seed, 0, count)


# ---- the engine bound to libspectre_b200.so -----------------------------------------------------------------------
class DeviceEngine:
    """Buffers are torch int64 tensors of shape (rows, 4) on the context's first device (PyTorch = device memory only).

    Stream contract (include/spectre_b200.h): every `_dev` entry point is ordered on the context's own stream and has
    completed when it returns. Every method below that makes torch allocate, zero, copy or assign runs with that stream
    (spb_stream) as torch's current stream, so the driver's memory traffic is in order with the library's kernels:
    no torch.cuda.synchronize() anywhere on the proof path (sync() exists for wall-clock laps)."""

    def __init__(self, backend, params, k, j):
        import torch
        self.torch, self.be, self.params, self.k, self.n = torch, backend, params, k, 1 << k
        self.dom = halo2.EvaluationDomain(backend, j, k)
        self.extended_k = self.dom.extended_k
        self.dev = torch.device("cuda", backend.devices[0])
        self.stream = torch.cuda.ExternalStream(backend.stream(0), device=self.dev)
        torch.cuda.synchronize(self.dev)                      # whatever the caller queued on other streams is complete

    # memory (all torch work on the context's stream)
    def alloc(self, rows):
        with self.torch.cuda.stream(self.stream):
            return self.torch.zeros((rows, 4), dtype=self.torch.int64, device=self.dev)
    def alloc_uninit(self, rows):
        """a buffer every element of which the next library call overwrites (extended cosets): no memset pass"""
        with self.torch.cuda.stream(self.stream):
            return self.torch.empty((rows, 4), dtype=self.torch.int64, device=self.dev)
    def upload(self, a):
        """host column -> device. A pinned torch tensor (witness buffers registered once by the caller) goes up as one
        asynchronous DMA; numpy arrays take the pageable path."""
        with self.torch.cuda.stream(self.stream):
            if isinstance(a, self.torch.Tensor):
                return a.view(self.torch.int64).reshape(-1, 4).to(self.dev, non_blocking=True)
            return self.torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to(self.dev)
    def download(self, b):
        with self.torch.cuda.stream(self.stream):
            return b.cpu().numpy().view(np.uint64)
    def clone(self, b):
        with self.torch.cuda.stream(self.stream):
            return b.clone()
    def view(self, b, lo, hi): return b[lo:hi]
    def write_rows(self, b, start, rows):
        rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, 4)
        if rows.shape[0]:
            with self.torch.cuda.stream(self.stream):
                b[start:start + rows.shape[0]] = self.upload(rows)
    def read_rows(self, b, start, count): return self.download(b[start:start + count])
    def random_rows(self, rows, generator=None):
        with self.torch.cuda.stream(self.stream):
            return uniform_residues(self.torch, rows, self.dev, generator)
    def random_chacha(self, seed, first, rows):
        """rows `Fr::random` draws number first.. of ChaCha20Rng::from_seed(seed), generated in HBM (spb_fr_random_chacha_dev)"""
        out = self.alloc_uninit(rows)
        self.be.fr_random_chacha_dev(seed, first, out.data_ptr(), rows)
        return out
    def sync(self): self.stream.synchronize()
    # proving-key file: polynomials go file <-> HBM through the library's double-buffered pinned staging, never through numpy
    def append_to_file(self, path, b, rows): self.be.write_file_dev(path, b.data_ptr(), rows * 32, append=True)
    def read_from_file(self, path, offset, rows):
        out = self.alloc_uninit(rows)
        self.be.read_file_dev(path, offset, out.data_ptr(), rows * 32)
        return out

    # commitments -> affine integer pairs
    def commit(self, basis, bufs, n):
        jac = self.params.commit_batch_dev(basis, [b.data_ptr() for b in bufs], n)
        return [halo2.jacobian_to_affine_ints(p) for p in jac]

    # domain
    def lagrange_to_coeff(self, b): self.dom.lagrange_to_coeff_dev(b.data_ptr())
    def lagrange_to_coeff_many(self, bufs):
        """in place; on a context with several devices the polynomials are spread over them (NTTs sharded by polynomial)"""
        if bufs:
            self.dom.lagrange_to_coeff_batch_dev([b.data_ptr() for b in bufs])
    def coeff_to_extended_many(self, bufs):
        outs = [self.alloc_uninit(1 << self.extended_k) for _ in bufs]
        if bufs:
            self.dom.coeff_to_extended_batch_dev([b.data_ptr() for b in bufs], [o.data_ptr() for o in outs])
        return outs
    def coeff_to_extended_part_many(self, bufs, part, outs):
        """outs[i] (n rows each) = rows part, part + R, ... of bufs[i]'s extended coset; the inputs are not written"""
        if bufs:
            self.dom.coeff_to_extended_part_batch_dev(part, [b.data_ptr() for b in bufs], [o.data_ptr() for o in outs])
    def extended_part_scatter(self, part_buf, part, values): self.dom.extended_part_scatter_dev(part, part_buf.data_ptr(), values.data_ptr())
    def zero(self, b):
        with self.torch.cuda.stream(self.stream):
            b.zero_()
    def coeff_to_lagrange(self, b):
        self.be.best_fft_dev(b.data_ptr(), fr_mont(omega_of(self.k)).reshape(1, 4), self.k)
    def coeff_to_extended(self, b):
        out = self.alloc_uninit(1 << self.extended_k)
        self.dom.coeff_to_extended_dev(b.data_ptr(), out.data_ptr())
        return out
    def extended_to_coeff(self, e, rows):
        out = self.alloc_uninit(rows)
        self.dom.extended_to_coeff_dev(e.data_ptr(), out.data_ptr())
        return out
    def divide_by_vanishing(self, e): self.dom.divide_by_vanishing_poly_dev(e.data_ptr())

    # quotient numerator
    def graph_evaluate(self, p, fixed, advice, instance, beta, gamma, theta, y, values, size, rot_scale):
        ptr = lambda bs: [b.data_ptr() for b in bs]
        self.be.graph_evaluate_dev(p["prog"], p["ncalc"], p["ncalc"], p["constants"], p["rotations"], ptr(fixed), ptr(advice), ptr(instance),
                                   np.zeros((1, 4), np.uint64), beta, gamma, theta, y, values.data_ptr(), size, rot_scale)
    def permutation_constraints(self, values, size, rot_scale, last_rotation, chunk_len, z, cols, sigma, l0, l_last, l_active, beta, gamma, y, ext_omega,
                                coset_generator=None):
        """X = zeta * ext_omega^idx at row idx, or coset_generator * ext_omega^idx when a generator is given (a coset part)"""
        ptr = lambda bs: [b.data_ptr() for b in bs]
        args = (values.data_ptr(), size, rot_scale, last_rotation, chunk_len, ptr(z), ptr(cols), ptr(sigma), l0.data_ptr(), l_last.data_ptr(), l_active.data_ptr(),
                beta, gamma, y)
        if coset_generator is None:
            self.be.permutation_constraints_dev(*args, ext_omega)
        else:
            self.be.permutation_constraints_coset_dev(*args, coset_generator, ext_omega)
    def lookup_constraints(self, values, size, rot_scale, product, pin, ptab, table_value, l0, l_last, l_active, beta, gamma, y):
        self.be.lookup_constraints_dev(values.data_ptr(), size, rot_scale, product.data_ptr(), pin.data_ptr(), ptab.data_ptr(), table_value.data_ptr(),
                                       l0.data_ptr(), l_last.data_ptr(), l_active.data_ptr(), beta, gamma, y)

    # argument provers
    def permute_expression_pair(self, a, s, usable, out_a, out_s):
        self.be.permute_expression_pair_dev(a.data_ptr(), s.data_ptr(), usable, out_a.data_ptr(), out_s.data_ptr())
    def permutation_product(self, values, sigma, first_col, beta, gamma, blinds, last_z, z):
        return self.be.permutation_product_dev(self.k, [b.data_ptr() for b in values], [b.data_ptr() for b in sigma], first_col, beta, gamma, blinds, last_z, z.data_ptr())
    def lookup_product(self, ci, ct, pi, pt, beta, gamma, blinds, z):
        self.be.lookup_product_dev(self.n, ci.data_ptr(), ct.data_ptr(), pi.data_ptr(), pt.data_ptr(), beta, gamma, blinds, z.data_ptr())

    # witness check
    def nonzero_rows(self, values, lo, hi, cap): return self.be.nonzero_rows_dev(values.data_ptr(), lo, hi, cap)
    def lookup_missing_rows(self, ci, ct, usable, cap): return self.be.lookup_missing_rows_dev(ci.data_ptr(), ct.data_ptr(), usable, cap)
    def copy_mismatches(self, values, sigma, usable, cap):
        return self.be.copy_mismatches_dev(self.k, [b.data_ptr() for b in values], [b.data_ptr() for b in sigma], usable, cap)

    # proving-key check
    def first_noncanonical(self, b, rows): return self.be.fr_first_noncanonical_dev(b.data_ptr(), rows)
    def sigma_check(self, sigma, usable, cap): return self.be.sigma_check_dev(self.k, [b.data_ptr() for b in sigma], usable, cap)
    def vec_axpy(self, y, alpha, x, n): self.be.vec_axpy_dev(y.data_ptr(), alpha, x.data_ptr(), n)

    # batch ops
    def eval_polynomial(self, b, n, point): return self.be.eval_polynomial_dev(b.data_ptr(), n, point)
    def eval_polynomial_many(self, pairs, n):
        out = self.be.eval_polynomial_many_dev([b.data_ptr() for b, _ in pairs], n, fr_mont_rows([pt for _, pt in pairs]))
        return [fr_int(r) for r in out]
    def lincomb(self, bufs, y, out, n): self.be.lincomb_dev([b.data_ptr() for b in bufs], y, out.data_ptr(), n)
    def vec_scale(self, b, alpha, n): self.be.vec_scale_dev(b.data_ptr(), alpha, n)

    # multi-open
    def shplonk_begin(self, sets, y, v):
        c, h = self.be.shplonk_begin_dev(self.params, self.n, [(pts, [b.data_ptr() for b in polys], ev) for pts, polys, ev in sets], y, v)
        return halo2.jacobian_to_affine_ints(c), h
    def shplonk_finish(self, state, u):
        return halo2.jacobian_to_affine_ints(self.be.shplonk_finish_dev(state, u))
    def shplonk_abort(self, state): self.be.shplonk_abort_dev(state)


def lagrange_to_coeff_many(E, bufs):
    """in place for every buffer; engines that can spread the transforms over several devices take the whole list"""
    if hasattr(E, "lagrange_to_coeff_many"):
        E.lagrange_to_coeff_many(list(bufs))
    else:
        for b in bufs:
            E.lagrange_to_coeff(b)


def eval_polynomial_many(E, pairs, n):
    """[(buffer, point:int)...] -> [eval:int...]; engines with a batched entry point evaluate the whole list in one launch"""
    if hasattr(E, "eval_polynomial_many"):
        return E.eval_polynomial_many(pairs, n)
    return [fr_int(E.eval_polynomial(buf, n, fr_mont(pt))) for buf, pt in pairs]


def coeff_to_extended_many(E, bufs):
    if hasattr(E, "coeff_to_extended_many"):
        return E.coeff_to_extended_many(list(bufs))
    return [E.coeff_to_extended(b) for b in bufs]


# ---- keygen -------------------------------------------------------------------------------------------------------
# Residency of a proving key's extended cosets (fixed, sigma, l0 / l_last / l_active: 2^extended_k rows each, about three
# quarters of a key's bytes). "resident" keeps them in device memory for the life of the key. "on_demand" (a lean key) keeps
# only the n-row data -- fixed / sigma values and polys, and the three l polynomials in coefficient form -- and create_proof
# rebuilds the cosets before the quotient and frees them after it. A rebuilt coset is the same coset, so the proof bytes are
# the same in both modes; a lean key costs one coset NTT per fixed / sigma / l column per proof.
# "per_part" holds what an on_demand key holds, and its proofs evaluate the quotient one coset part at a time: the extended
# rows part + R m (m < n, R = 2^(extended_k - k)) of every column are built as n-row buffers, evaluated and scattered into the
# one extended `values`, so no column but `values` and the quotient's coefficients ever has more than n rows. It trades more,
# smaller transforms for a peak that is about one extended buffer instead of one per column; the proof bytes are the same.
COSETS_MODES = ("resident", "on_demand", "per_part")


class ProvingKey:
    """A lean key (cosets="on_demand" or "per_part") has fixed_cosets = sigma_cosets = l0 = l_last = l_active = None and holds
    `l_polys` = [l0, l_last, l_active] in coefficient form instead (None in a resident key)."""

    per_part = False                                         # cosets="per_part": create_proof evaluates the quotient per coset part

    @property
    def lean(self):
        return self.fixed_cosets is None


def key_device_bytes(cs, k, extended_k, cosets="resident"):
    """Device bytes a proving key of this shape holds (DESIGN.md section 3), with C = num_fixed + len(permutation) columns:
    32 * (2 C 2^k + (C + 3) 2^extended_k) resident, 32 * (2 C + 3) 2^k lean (on_demand and per_part)."""
    _check_cosets_mode(cosets)
    cols = cs.num_fixed + len(cs.permutation)
    if cosets == "resident":
        return 32 * ((2 * cols << k) + ((cols + 3) << extended_k))
    return 32 * ((2 * cols + 3) << k)


def _check_cosets_mode(cosets):
    if cosets not in COSETS_MODES:
        raise ValueError("cosets must be one of %s, not %r" % (", ".join(COSETS_MODES), cosets))


def l_polys(E, n, usable_rows):
    """[l0, l_last, l_active] in coefficient form: l_active = 1 - l_last - l_blind is one on the rows [0, usable_rows)"""
    one = fr_mont(1).reshape(1, 4)
    l0 = E.alloc(n); E.write_rows(l0, 0, one)
    l_last = E.alloc(n); E.write_rows(l_last, usable_rows, one)
    l_active = E.alloc(n); E.write_rows(l_active, 0, np.broadcast_to(one, (usable_rows, 4)))
    ls = [l0, l_last, l_active]
    lagrange_to_coeff_many(E, ls)
    return ls


def build_sigma(E, cs, k, copies):
    """permutation::keygen::Assembly::build_pk: sigma_c[i] = delta^c' * omega^i' of the cell (c', i') that follows
    (c, i) in its copy cycle. `copies`: list of ((col, row), (col, row)) equalities between permutation columns.
    The identity columns delta^c * omega^i are produced on the device (one NTT of X, then scalings); only the cells on
    non-trivial cycles are patched from the host."""
    n = 1 << k
    n_cols = len(cs.permutation)
    x_poly = np.zeros((n, 4), dtype=np.uint64); x_poly[1] = fr_mont(1)
    base = E.upload(x_poly)
    E.coeff_to_lagrange(base)                               # omega^i
    sigma = []
    for c in range(n_cols):
        s = E.clone(base)
        if c:
            E.vec_scale(s, fr_mont(pow(DELTA, c, R_MOD)), n)
        sigma.append(s)
    # union the copies into cycles (halo2 keeps mapping / aux / sizes arrays; same resulting cycles up to rotation,
    # and any cyclic order of a class yields a valid sigma -- the order below is insertion order)
    nxt = {}
    def cell_next(c): return nxt.get(c, c)
    def cycle_of(c):
        out, cur = [c], cell_next(c)
        while cur != c:
            out.append(cur); cur = cell_next(cur)
        return out
    for a, b in copies:
        if b in cycle_of(a):
            continue
        na, nb = cell_next(a), cell_next(b)                 # splice the two cycles
        nxt[a], nxt[b] = nb, na
    w = omega_of(k)
    for (c, i), (c2, i2) in nxt.items():
        E.write_rows(sigma[c], i, fr_mont(pow(DELTA, c2, R_MOD) * pow(w, i2, R_MOD)).reshape(1, 4))
    return sigma


def keygen(E, cs, k, fixed_columns, copies, vk_digest=None, cosets="resident"):
    """keygen_vk + keygen_pk: fixed and sigma commitments, their coefficient forms and extended cosets, l0 / l_last /
    l_active cosets -- all left resident on the device. fixed_columns: list of (n, 4) Montgomery arrays (Lagrange).
    cosets="on_demand" makes a lean key: no coset is ever computed, create_proof rebuilds them for each proof.
    cosets="per_part" makes the same lean key, whose proofs build the cosets one n-row part at a time."""
    _check_cosets_mode(cosets)
    n = 1 << k
    pk = ProvingKey()
    pk.cs, pk.k, pk.n = cs, k, n
    pk.per_part = cosets == "per_part"
    bf = cs.blinding_factors()
    pk.blinding_factors, pk.usable_rows = bf, n - (bf + 1)
    pk.fixed_values = [E.upload(c) for c in fixed_columns]
    pk.sigma_values = build_sigma(E, cs, k, copies)
    G_LAG = halo2.BASIS_G_LAGRANGE
    pk.fixed_commitments = E.commit(G_LAG, pk.fixed_values, n) if pk.fixed_values else []
    pk.sigma_commitments = E.commit(G_LAG, pk.sigma_values, n) if pk.sigma_values else []

    def polys(values):
        ps = [E.clone(v) for v in values]
        lagrange_to_coeff_many(E, ps)
        return ps
    pk.fixed_polys, pk.sigma_polys = polys(pk.fixed_values), polys(pk.sigma_values)
    ls = l_polys(E, n, pk.usable_rows)
    if cosets == "resident":
        pk.fixed_cosets = coeff_to_extended_many(E, pk.fixed_polys)
        pk.sigma_cosets = coeff_to_extended_many(E, pk.sigma_polys)
        pk.l0, pk.l_last, pk.l_active = coeff_to_extended_many(E, ls)
        pk.l_polys = None
    else:
        pk.fixed_cosets = pk.sigma_cosets = pk.l0 = pk.l_last = pk.l_active = None
        pk.l_polys = ls
    pk.vk_digest = vk_digest if vk_digest is not None else default_vk_digest(pk)
    return pk


def default_vk_digest(pk):
    """Stand-in for VerifyingKey::transcript_repr (upstream: a Blake2b hash of the pinned VK's debug format, which cannot
    be reproduced without the Rust types): Keccak over k and the VK commitments."""
    from .transcript import keccak256
    data = bytearray(pk.k.to_bytes(4, "little"))
    for x, y in pk.fixed_commitments + pk.sigma_commitments:
        data += x.to_bytes(32, "big") + y.to_bytes(32, "big")
    return int.from_bytes(keccak256(bytes(data)), "big") % R_MOD


# ---- ProvingKey::write / ::read (SerdeFormat::RawBytesUnchecked) ------------------------------------------------------------
# Layout of [UPSTREAM] halo2_proofs/src/plonk.rs `ProvingKey::write` as Spectre stores it (`*.pkey`, read at start-up by
# ProverState::new, prover/src/prover.rs:44-116, through lightclient-circuits/src/util/circuit.rs:104-115,273-280):
#   VerifyingKey:  k (u32 BE) | #fixed commitments (u32 BE) | fixed commitments | permutation commitments | selectors
#                  (none here: the shapes of this repo keep selectors as fixed columns, compress_selectors = false)
#   l0 | l_last | l_active                          each a Polynomial: len (u32 BE) | values
#   fixed_values | fixed_polys | fixed_cosets        each a slice: count (u32 BE) | Polynomial...
#   permutation::ProvingKey: permutations | polys | cosets    (three slices)
# Field elements and curve coordinates are their in-memory Montgomery limbs (RawBytes). The constraint system is not in the
# file: like upstream's `ProvingKey::read::<_, ConcreteCircuit>(reader, format, params)` the reader gets it from the circuit.
# This restates the upstream layout from memory (no Rust toolchain here to diff a real .pkey against it): files written and
# read by this repo round-trip, byte compatibility with upstream's files is unverified.
_FQ_MONT = (1 << 256) % P_MOD


def _point_bytes(pt):
    x, y = pt
    return b"".join(((v * _FQ_MONT) % P_MOD).to_bytes(32, "little") for v in (x, y))


def _point_from(raw):
    inv = pow(_FQ_MONT, -1, P_MOD)
    return tuple(int.from_bytes(raw[i:i + 32], "little") * inv % P_MOD for i in (0, 32))


def write_pk(E, pk, path):
    """ProvingKey::write(writer, SerdeFormat::RawBytesUnchecked): header and commitments from the host, every polynomial
    streamed from device memory by the engine. A lean key writes the same bytes: each coset is rebuilt into one temporary
    buffer, appended and freed before the next."""
    with open(path, "wb") as f:
        f.write(pk.k.to_bytes(4, "big") + len(pk.fixed_commitments).to_bytes(4, "big"))
        for pt in pk.fixed_commitments + pk.sigma_commitments:
            f.write(_point_bytes(pt))

    def poly(b, rows):
        with open(path, "ab") as f:
            f.write(rows.to_bytes(4, "big"))
        E.append_to_file(path, b, rows)

    def polys(bufs, rows, count):
        with open(path, "ab") as f:
            f.write(count.to_bytes(4, "big"))
        for b in bufs:
            poly(b, rows)
            del b                                            # a rebuilt coset is freed before the next one is built

    def cosets(resident, coeffs):
        return resident if resident is not None else (E.coeff_to_extended(p) for p in coeffs)
    ext = 1 << E.extended_k
    for b in cosets(None if pk.lean else [pk.l0, pk.l_last, pk.l_active], pk.l_polys):
        poly(b, ext)
        del b
    nf, m = len(pk.fixed_polys), len(pk.sigma_polys)
    polys(pk.fixed_values, pk.n, nf); polys(pk.fixed_polys, pk.n, nf); polys(cosets(pk.fixed_cosets, pk.fixed_polys), ext, nf)
    polys(pk.sigma_values, pk.n, m); polys(pk.sigma_polys, pk.n, m); polys(cosets(pk.sigma_cosets, pk.sigma_polys), ext, m)


PK_FORMATS = ("RawBytes", "RawBytesUnchecked")


def _point_check(raw):
    """None for a G1Affine as RawBytes stores it that halo2curves' checked read accepts (canonical coordinates on y^2 = x^3 + 3,
    or the identity (0, 0)), else the reason it is refused (the texts of the params check, spb_srs_read_file_custom)"""
    rx, ry = int.from_bytes(raw[:32], "little"), int.from_bytes(raw[32:64], "little")
    if rx >= P_MOD:
        return "x is not less than the field modulus"
    if ry >= P_MOD:
        return "y is not less than the field modulus"
    if rx == 0 and ry == 0:
        return None
    x, y = _point_from(raw)
    return None if (y * y - x * x * x - 3) % P_MOD == 0 else "not on the curve"


def read_pk(E, cs, path, vk_digest=None, cosets="resident", format="RawBytesUnchecked"):
    """ProvingKey::read: the inverse of write_pk; `cs` plays the role of the concrete circuit's configure().
    cosets="on_demand" reads a lean key from the same file: the coset sections are skipped, never read, and the three l
    polynomials are rebuilt from their definition. cosets="per_part" reads the same lean key for per-part proofs.

    format="RawBytesUnchecked" (SerdeFormat::RawBytesUnchecked) believes every byte. format="RawBytes" is upstream's checked
    read: every VK point is checked on the host (coordinates below p, on the curve or the identity) and every polynomial is
    scanned on the device right after it lands (spb_fr_first_noncanonical_dev: limbs below r). The first failure in file order
    raises ValueError naming the file, the section and index, the row and the reason; the buffers already read are freed. A
    lean read never reads the coset sections, so it does not check them either. The read says nothing about whether the key
    belongs to the params it is used with: that is check_pk."""
    _check_cosets_mode(cosets)
    if format not in PK_FORMATS:
        raise ValueError("read_pk: format must be one of %s (the compressed Processed format is not implemented)" % sorted(PK_FORMATS))
    checked = format == "RawBytes"
    lean = cosets != "resident"
    pk = ProvingKey()
    pk.per_part = cosets == "per_part"
    with open(path, "rb") as f:
        head = f.read(8)
        k, n_fixed = int.from_bytes(head[:4], "big"), int.from_bytes(head[4:], "big")
        if k != E.k or n_fixed != cs.num_fixed:
            raise ValueError("read_pk: %s is for k = %d with %d fixed columns, expected k = %d with %d" % (path, k, n_fixed, E.k, cs.num_fixed))
        raws = [f.read(64) for _ in range(n_fixed + len(cs.permutation))]
        pos = [f.tell()]
        size = f.seek(0, 2)
    if checked:
        for i, raw in enumerate(raws):
            why = _point_check(raw)
            if why is not None:
                what = "fixed commitment %d" % i if i < n_fixed else "sigma commitment %d" % (i - n_fixed)
                raise ValueError("read_pk: %s: %s: %s" % (path, what, why))
    pts = [_point_from(raw) for raw in raws]
    n, ext = 1 << k, 1 << E.extended_k
    pk.cs, pk.k, pk.n = cs, k, n
    pk.blinding_factors = cs.blinding_factors(); pk.usable_rows = n - (pk.blinding_factors + 1)
    pk.fixed_commitments, pk.sigma_commitments = pts[:n_fixed], pts[n_fixed:]

    def u32():
        with open(path, "rb") as f:
            f.seek(pos[0]); v = int.from_bytes(f.read(4), "big")
        pos[0] += 4
        return v

    def poly(rows, what, skip=False):
        if u32() != rows:
            raise ValueError("read_pk: polynomial length mismatch in %s" % path)
        b = None if skip else E.read_from_file(path, pos[0], rows)
        pos[0] += rows * 32
        if checked and b is not None:
            bad = E.first_noncanonical(b, rows)
            if bad < rows:
                del b
                raise ValueError("read_pk: %s: %s row %d: not a canonical field element" % (path, what, bad))
        return b

    def polys(count, rows, what, skip=False):
        if u32() != count:
            raise ValueError("read_pk: slice length mismatch in %s" % path)
        bufs = [poly(rows, "%s[%d]" % (what, i), skip) for i in range(count)]
        return None if skip else bufs
    m = len(cs.permutation)
    try:
        pk.l0, pk.l_last, pk.l_active = poly(ext, "l0", lean), poly(ext, "l_last", lean), poly(ext, "l_active", lean)
        pk.fixed_values, pk.fixed_polys = polys(n_fixed, n, "fixed_values"), polys(n_fixed, n, "fixed_polys")
        pk.fixed_cosets = polys(n_fixed, ext, "fixed_cosets", lean)
        pk.sigma_values, pk.sigma_polys = polys(m, n, "sigma_values"), polys(m, n, "sigma_polys")
        pk.sigma_cosets = polys(m, ext, "sigma_cosets", lean)
    except ValueError:
        pk.__dict__.clear()                                  # the buffers already read are freed, even while the error is held
        raise
    if pos[0] != size:
        raise ValueError("read_pk: %d trailing bytes in %s" % (size - pos[0], path))
    pk.l_polys = l_polys(E, n, pk.usable_rows) if lean else None
    pk.vk_digest = vk_digest if vk_digest is not None else default_vk_digest(pk)
    return pk


# ---- multi-open bookkeeping ---------------------------------------------------------------------------------------
def rotation_sets(queries_):
    """construct_intermediate_sets: queries = [(poly_id, point:int, eval:int)] in query order ->
    [(points sorted as Fr's Ord, [poly_id...], evals[poly][point])], sets and polynomials in first-seen order."""
    per_poly, order = {}, []
    for pid, pt, _ in queries_:
        if pid not in per_poly:
            per_poly[pid] = set(); order.append(pid)
        per_poly[pid].add(pt)
    sets = []
    for pid in order:
        key = frozenset(per_poly[pid])
        for s in sets:
            if s[0] == key:
                s[1].append(pid); break
        else:
            sets.append((key, [pid]))
    out = []
    for key, pids in sets:
        pts = sorted(key)
        evals = [[next(ev for p2, pt2, ev in queries_ if p2 == pid and pt2 == pt) for pt in pts] for pid in pids]
        out.append((pts, pids, evals))
    return out


# ---- create_proof -------------------------------------------------------------------------------------------------
def evaluate_h_per_part(E, pk, advice_polys, inst_polys, perm_polys, lookups, beta, gamma, theta, y, lap):
    """Evaluator::evaluate_h one coset part at a time (a per-part key); returns the extended `values` (2^extended_k rows).
    Part j < R = 2^(extended_k - k) is the extended rows j + R m, m < n: the values at g_j omega^m with g_j = zeta
    extended_omega^j. A rotation by r reads row (m + r) mod n of the same part, so the gate, permutation and lookup passes run
    on a part with size n and rot_scale 1; only the permutation argument, which reads X itself, takes g_j. Every extended row
    sees the same field operations in the same order as in the whole-coset evaluation, so `values` is the same.
    Every part buffer is allocated once per proof and freed when this returns, before divide_by_vanishing."""
    cs, k, n = pk.cs, pk.k, pk.n
    R = 1 << (E.extended_k - k)
    bf = pk.blinding_factors
    ext_omega = pow(ROOT_OF_UNITY, 1 << (28 - E.extended_k), R_MOD)
    omega = fr_mont(omega_of(k))
    srcs = pk.fixed_polys + pk.sigma_polys + pk.l_polys + advice_polys + inst_polys + perm_polys
    for L in lookups:
        srcs += [L.product_poly, L.permuted_input_poly, L.permuted_table_poly]
    parts = [E.alloc(n) for _ in srcs]
    at = [0]

    def take(count):
        at[0] += count
        return parts[at[0] - count:at[0]]
    fixed_p, sigma_p, (l0, l_last, l_active) = take(len(pk.fixed_polys)), take(len(pk.sigma_polys)), take(3)
    advice_p, inst_p, z_p = take(len(advice_polys)), take(len(inst_polys)), take(len(perm_polys))
    lookup_p = [take(3) for _ in lookups]
    cols = [{"fixed": fixed_p, "advice": advice_p, "instance": inst_p}[kind][c] for kind, c in cs.permutation]
    gates = cs.gates_program() if cs.gates else None
    table_programs = [cs.lookup_value_program(li) for li in range(len(lookups))]
    part_values = E.alloc(n)
    table_value = E.alloc(n) if lookups else None
    values = E.alloc(1 << E.extended_k)
    zero4 = fr_mont(0)
    for j in range(R):
        E.coeff_to_extended_part_many(srcs, j, parts)
        lap("coeff_to_extended")
        if j:
            E.zero(part_values)                              # PreviousValue of the gates reads it: every part starts at zero
        if gates is not None:
            E.graph_evaluate(gates, fixed_p, advice_p, inst_p, beta, gamma, theta, y, part_values, n, 1)
        if perm_polys:
            g = fr_mont(ZETA * pow(ext_omega, j, R_MOD))
            E.permutation_constraints(part_values, n, 1, -(bf + 1), cs.chunk_len(), z_p, cols, sigma_p, l0, l_last, l_active, beta, gamma, y, omega,
                                      coset_generator=g)
        for li, (pc, ic, tc) in enumerate(lookup_p):
            if j or li:
                E.zero(table_value)
            E.graph_evaluate(table_programs[li], fixed_p, advice_p, inst_p, beta, gamma, theta, zero4, table_value, n, 1)
            E.lookup_constraints(part_values, n, 1, pc, ic, tc, table_value, l0, l_last, l_active, beta, gamma, y)
        E.extended_part_scatter(part_values, j, values)
        lap("evaluate_h")
    return values


def create_proof(E, pk, instances, advice_columns, rng, transcript, timings=None):
    """halo2_proofs::plonk::create_proof for one circuit over KZG/SHPLONK (single phase, no challenges API).
    instances: per instance column a list of ints; advice_columns: per advice column an (n, 4) Montgomery array whose
    rows >= usable_rows are overwritten with blinding; rng(count) -> (count, 4) Montgomery draws, consumed in
    upstream's order; transcript: EvmTranscriptWrite-like. Returns the proof bytes."""
    import time
    cs, k, n = pk.cs, pk.k, pk.n
    bf, usable = pk.blinding_factors, pk.usable_rows
    ext_n, rot_scale = 1 << E.extended_k, 1 << (E.extended_k - k)
    G, GL = halo2.BASIS_G, halo2.BASIS_G_LAGRANGE
    w = omega_of(k)
    t_last = [time.perf_counter()]

    def lap(name):
        if timings is not None:
            E.sync(); t = time.perf_counter(); timings[name] = timings.get(name, 0.0) + t - t_last[0]; t_last[0] = t

    # 1. vk, instances
    if len(instances) != cs.num_instance:
        raise ValueError("create_proof: %d instance columns given, the circuit has %d (upstream: Error::InvalidInstances)" % (len(instances), cs.num_instance))
    if len(advice_columns) != cs.num_advice:
        raise ValueError("create_proof: %d advice columns given, the circuit has %d" % (len(advice_columns), cs.num_advice))
    for col in instances:
        for v in col:
            transcript.common_scalar(v)                      # KZG: instances enter the transcript, no commitments
    inst_values = []
    for col in instances:
        if len(col) > usable:
            raise ValueError("create_proof: an instance column has more than %d values (upstream: Error::InstanceTooLarge)" % usable)
        b = E.alloc(n); E.write_rows(b, 0, fr_mont_rows(col)); inst_values.append(b)
    inst_polys = [E.clone(b) for b in inst_values]
    lagrange_to_coeff_many(E, inst_polys)
    lap("instances")

    # 2. advice: blind the unusable rows, commit, to coefficient form
    advice_values = []
    for col in advice_columns:
        b = E.upload(col)
        E.write_rows(b, usable, rng(bf + 1))
        advice_values.append(b)
    rng(len(advice_values))                                  # Blind(random) per column: unused by KZG, drawn upstream
    for pt in E.commit(GL, advice_values, n):
        transcript.write_ec_point(pt)
    advice_polys = [E.clone(b) for b in advice_values]
    lagrange_to_coeff_many(E, advice_polys)
    lap("advice")

    theta = fr_mont(transcript.squeeze_challenge())
    zero4 = fr_mont(0)

    # 3. lookups: compress, permute, commit
    class _L: pass
    lookups = []
    for ins, tbs in cs.lookups:
        L = _L()
        L.compressed_input, L.compressed_table = E.alloc(n), E.alloc(n)
        E.graph_evaluate(cs.lookup_compress_program(ins), pk.fixed_values, advice_values, inst_values, zero4, zero4, theta, zero4, L.compressed_input, n, 1)
        E.graph_evaluate(cs.lookup_compress_program(tbs), pk.fixed_values, advice_values, inst_values, zero4, zero4, theta, zero4, L.compressed_table, n, 1)
        L.permuted_input, L.permuted_table = E.alloc(n), E.alloc(n)
        E.permute_expression_pair(L.compressed_input, L.compressed_table, usable, L.permuted_input, L.permuted_table)
        E.write_rows(L.permuted_input, usable, rng(bf + 1))
        E.write_rows(L.permuted_table, usable, rng(bf + 1))
        rng(2)                                               # the two commitment blinds
        for pt in E.commit(GL, [L.permuted_input, L.permuted_table], n):
            transcript.write_ec_point(pt)
        L.permuted_input_poly, L.permuted_table_poly = E.clone(L.permuted_input), E.clone(L.permuted_table)
        lagrange_to_coeff_many(E, [L.permuted_input_poly, L.permuted_table_poly])
        lookups.append(L)
    lap("lookup_permuted")

    beta = fr_mont(transcript.squeeze_challenge())
    gamma = fr_mont(transcript.squeeze_challenge())

    # 4. permutation grand products, one per chunk of columns
    col_values = [{"fixed": pk.fixed_values, "advice": advice_values, "instance": inst_values}[kind][c] for kind, c in cs.permutation]
    chunk = cs.chunk_len()                                   # degree() >= 3, so >= 1
    perm_z, last_z = [], fr_mont(1)
    for lo in range(0, len(col_values), chunk):
        hi = min(lo + chunk, len(col_values))
        z = E.alloc(n)
        last_z = E.permutation_product(col_values[lo:hi], pk.sigma_values[lo:hi], lo, beta, gamma, rng(bf), last_z, z)
        rng(1)
        perm_z.append(z)
    if perm_z:
        for pt in E.commit(GL, perm_z, n):
            transcript.write_ec_point(pt)
    perm_polys = perm_z                                      # converted in place: the Lagrange form is not needed again
    lagrange_to_coeff_many(E, perm_polys)
    lap("permutation_product")

    # 5. lookup grand products
    for L in lookups:
        L.product = E.alloc(n)
        E.lookup_product(L.compressed_input, L.compressed_table, L.permuted_input, L.permuted_table, beta, gamma, rng(bf), L.product)
        rng(1)
    if lookups:
        for pt in E.commit(GL, [L.product for L in lookups], n):
            transcript.write_ec_point(pt)
    lagrange_to_coeff_many(E, [L.product for L in lookups])
    for L in lookups:
        L.product_poly = L.product
        L.compressed_input = L.compressed_table = L.permuted_input = L.permuted_table = None
    lap("lookup_product")

    # 6. vanishing argument: random polynomial
    # an rng that offers device_rows(E, count) draws the n coefficients on the device; otherwise they come from the host stream
    random_poly = rng.device_rows(E, n) if hasattr(rng, "device_rows") else E.upload(rng(n))
    rng(1)
    transcript.write_ec_point(E.commit(G, [random_poly], n)[0])
    lap("vanishing_commit")

    y = fr_mont(transcript.squeeze_challenge())

    # 7. quotient: extended cosets, evaluate_h, divide by the vanishing polynomial, split, commit
    # a lean key's cosets are rebuilt here and freed with the advice cosets, before divide_by_vanishing; a per-part key's
    # proof builds every coset one n-row part at a time (evaluate_h_per_part)
    if pk.per_part:
        values = evaluate_h_per_part(E, pk, advice_polys, inst_polys, perm_polys, lookups, beta, gamma, theta, y, lap)
    else:
        if pk.lean:
            nf, ns = len(pk.fixed_polys), len(pk.sigma_polys)
            key = coeff_to_extended_many(E, pk.fixed_polys + pk.sigma_polys + pk.l_polys)
            fixed_cosets, sigma_cosets, (l0, l_last, l_active) = key[:nf], key[nf:nf + ns], key[nf + ns:]
            del key
            lap("key_cosets")
        else:
            fixed_cosets, sigma_cosets, l0, l_last, l_active = pk.fixed_cosets, pk.sigma_cosets, pk.l0, pk.l_last, pk.l_active
        both = coeff_to_extended_many(E, advice_polys + inst_polys)
        advice_cosets, inst_cosets = both[:len(advice_polys)], both[len(advice_polys):]
        del both
        lap("coeff_to_extended")
        values = E.alloc(ext_n)
        if cs.gates:
            E.graph_evaluate(cs.gates_program(), fixed_cosets, advice_cosets, inst_cosets, beta, gamma, theta, y, values, ext_n, rot_scale)
        if perm_polys:
            z_cosets = coeff_to_extended_many(E, perm_polys)
            cosets = [{"fixed": fixed_cosets, "advice": advice_cosets, "instance": inst_cosets}[kind][c] for kind, c in cs.permutation]
            ext_omega = fr_mont(pow(ROOT_OF_UNITY, 1 << (28 - E.extended_k), R_MOD))
            E.permutation_constraints(values, ext_n, rot_scale, -(bf + 1), chunk, z_cosets, cosets, sigma_cosets, l0, l_last, l_active, beta, gamma, y, ext_omega)
            del z_cosets, cosets
        for li, L in enumerate(lookups):
            table_value = E.alloc(ext_n)
            E.graph_evaluate(cs.lookup_value_program(li), fixed_cosets, advice_cosets, inst_cosets, beta, gamma, theta, zero4, table_value, ext_n, rot_scale)
            pc, ic, tc = coeff_to_extended_many(E, [L.product_poly, L.permuted_input_poly, L.permuted_table_poly])
            E.lookup_constraints(values, ext_n, rot_scale, pc, ic, tc, table_value, l0, l_last, l_active, beta, gamma, y)
            del table_value, pc, ic, tc
        del advice_cosets, inst_cosets, fixed_cosets, sigma_cosets, l0, l_last, l_active
        lap("evaluate_h")
    E.divide_by_vanishing(values)
    pieces_n = cs.degree() - 1
    h_coeff = E.extended_to_coeff(values, n * pieces_n)
    del values
    h_pieces = [E.view(h_coeff, i * n, (i + 1) * n) for i in range(pieces_n)]
    rng(pieces_n)
    for pt in E.commit(G, h_pieces, n):
        transcript.write_ec_point(pt)
    lap("vanishing_construct")

    x = transcript.squeeze_challenge()
    xm = fr_mont(x)
    x_pow = lambda rot: x * pow(w, rot % n, R_MOD) % R_MOD

    # 8. evaluations, in the order the verifier reads them. Every (polynomial, point) query is collected first and evaluated by
    # ONE engine call (one kernel launch for the whole list), then the scalars enter the transcript in upstream's order.
    polys, evals_q, todo = {}, [], []                        # poly id -> buffer; [(poly id, point, eval)] in multi-open order

    def ask(pid, buf, rot):
        polys[pid] = buf
        todo.append((buf, x_pow(rot)))
        return len(todo) - 1

    adv_i = [ask(("advice", c), advice_polys[c], r) for c, r in cs.advice_queries]
    fix_i = [ask(("fixed", c), pk.fixed_polys[c], r) for c, r in cs.fixed_queries]
    # vanishing::evaluate: h(X) = sum_i x^(n i) h_i(X), and the random polynomial at x
    h_poly = E.alloc(n)
    E.lincomb(h_pieces, fr_mont(pow(x, n, R_MOD)), h_poly, n)
    rnd_i = ask(("random",), random_poly, 0)
    sig_i = [ask(("sigma", c), pk.sigma_polys[c], 0) for c in range(len(pk.sigma_polys))]
    perm_i = [(ask(("perm", s), p, 0), ask(("perm", s), p, 1), ask(("perm", s), p, -(bf + 1)) if s + 1 < len(perm_polys) else None)
              for s, p in enumerate(perm_polys)]
    look_i = [(ask(("lk_z", li), L.product_poly, 0), ask(("lk_z", li), L.product_poly, 1), ask(("lk_a", li), L.permuted_input_poly, 0),
               ask(("lk_a", li), L.permuted_input_poly, -1), ask(("lk_s", li), L.permuted_table_poly, 0)) for li, L in enumerate(lookups)]
    h_i = ask(("h",), h_poly, 0)
    values = eval_polynomial_many(E, todo, n)
    got = lambda i: None if i is None else (todo[i][1], values[i])
    adv_e, fix_e, rnd_e, sig_e = [got(i) for i in adv_i], [got(i) for i in fix_i], got(rnd_i), [got(i) for i in sig_i]
    perm_e = [tuple(got(i) for i in t) for t in perm_i]
    look_e = [tuple(got(i) for i in t) for t in look_i]
    for _, e in adv_e: transcript.write_scalar(e)
    for _, e in fix_e: transcript.write_scalar(e)
    transcript.write_scalar(rnd_e[1])
    for _, e in sig_e: transcript.write_scalar(e)
    for e0, e1, el in perm_e:
        transcript.write_scalar(e0[1]); transcript.write_scalar(e1[1])
        if el is not None:
            transcript.write_scalar(el[1])
    for t in look_e:
        for _, e in t: transcript.write_scalar(e)
    lap("evaluations")

    # 9. multi-open queries in create_proof's order: advice, permutation z, lookups, fixed, sigma, vanishing
    for (c, r), (pt, e) in zip(cs.advice_queries, adv_e): evals_q.append((("advice", c), pt, e))
    for s, (e0, e1, _) in enumerate(perm_e):
        evals_q.append((("perm", s), e0[0], e0[1])); evals_q.append((("perm", s), e1[0], e1[1]))
    for s in reversed(range(len(perm_e) - 1)):
        el = perm_e[s][2]; evals_q.append((("perm", s), el[0], el[1]))
    for li, (pe, pne, ie, iie, te) in enumerate(look_e):
        evals_q += [(("lk_z", li), pe[0], pe[1]), (("lk_a", li), ie[0], ie[1]), (("lk_s", li), te[0], te[1]), (("lk_a", li), iie[0], iie[1]), (("lk_z", li), pne[0], pne[1])]
    for (c, r), (pt, e) in zip(cs.fixed_queries, fix_e): evals_q.append((("fixed", c), pt, e))
    for c, (pt, e) in enumerate(sig_e): evals_q.append((("sigma", c), pt, e))
    h_eval = got(h_i)[1]
    evals_q.append((("h",), x, h_eval)); evals_q.append((("random",), rnd_e[0], rnd_e[1]))

    sets = [(fr_mont_rows(pts), [polys[p] for p in pids], np.stack([fr_mont_rows(row) for row in evs])) for pts, pids, evs in rotation_sets(evals_q)]
    y2 = fr_mont(transcript.squeeze_challenge())
    v = fr_mont(transcript.squeeze_challenge())
    h1, state = E.shplonk_begin(sets, y2, v)
    try:
        transcript.write_ec_point(h1)
        u = fr_mont(transcript.squeeze_challenge())
    except BaseException:                                     # KeyboardInterrupt too: an open handle holds the context's workspace
        E.shplonk_abort(state)
        raise
    transcript.write_ec_point(E.shplonk_finish(state, u))    # finish consumes the handle, also when it raises
    lap("shplonk")
    return bytes(transcript.proof)


# ---- witness check ------------------------------------------------------------------------------------------------
class WitnessFailure(namedtuple("WitnessFailure", "kind index rows total mapped", defaults=(None,))):
    """One failing constraint of check_witness. kind: "gate" (index = the gate's position in cs.gates), "lookup" (its
    position in cs.lookups) or "copy" (the permutation column's position in cs.permutation); rows: the first failing rows,
    ascending; total: how many rows fail; mapped: for "copy", the (column, row) each of `rows` is copied to (else None)."""


def check_witness(E, pk, instances, advice_columns, theta=None, max_rows=16):
    """halo2_proofs::dev::MockProver::verify on the engine: every constraint the witness fails, as a list of WitnessFailure in
    the order gates, lookups, permutation columns; [] for a satisfied witness. Nothing is written to the key, and the
    caller's columns are uploaded as they are (no blinding rows are drawn), so it can run before or instead of create_proof.

    With u = pk.usable_rows and n = 2^k, every read is of the n-row Lagrange values, rotations wrapping mod n:
      * a gate must evaluate to zero at every row i < u (a rotated read into the rows >= u reads what the caller put there);
      * a lookup's input tuple at every row i < u must equal its table tuple at some row j < u. Both sides are compressed with
        a random theta as create_proof compresses them (theta=None draws it from `secrets`); a tuple that is in no table row
        passes only if its compression collides with one of the u table values, probability about u / r for the field size r;
      * at every row i < u of permutation column c, the cell must hold the value of the cell (c', i') that sigma_c[i] labels.
    Instances are laid out as create_proof lays them out. A key whose sigma labels a cell outside the usable rows raises the
    engine's error naming the column and row."""
    cs, n, usable = pk.cs, pk.n, pk.usable_rows
    if len(instances) != cs.num_instance:
        raise ValueError("check_witness: %d instance columns given, the circuit has %d (upstream: Error::InvalidInstances)" % (len(instances), cs.num_instance))
    if len(advice_columns) != cs.num_advice:
        raise ValueError("check_witness: %d advice columns given, the circuit has %d" % (len(advice_columns), cs.num_advice))
    inst_values = []
    for col in instances:
        if len(col) > usable:
            raise ValueError("check_witness: an instance column has more than %d values (upstream: Error::InstanceTooLarge)" % usable)
        b = E.alloc(n); E.write_rows(b, 0, fr_mont_rows(col)); inst_values.append(b)
    advice_values = [E.upload(col) for col in advice_columns]
    fixed = pk.fixed_values
    zero4 = fr_mont(0)
    failures = []
    if cs.gates:
        values = E.alloc(n)
        for g, gate in enumerate(cs.gates):
            p = Program()
            p.horner(p._const(0), p._const(0), [gate])           # 0 * 0 + gate: this gate alone, no y-folding
            E.graph_evaluate(p.finish(), fixed, advice_values, inst_values, zero4, zero4, zero4, zero4, values, n, 1)
            rows, total = E.nonzero_rows(values, 0, usable, max_rows)
            if total:
                failures.append(WitnessFailure("gate", g, rows, total))
    theta = fr_mont(secrets.randbelow(R_MOD) if theta is None else theta)
    for li, (ins, tbs) in enumerate(cs.lookups):
        ci, ct = E.alloc(n), E.alloc(n)
        E.graph_evaluate(cs.lookup_compress_program(ins), fixed, advice_values, inst_values, zero4, zero4, theta, zero4, ci, n, 1)
        E.graph_evaluate(cs.lookup_compress_program(tbs), fixed, advice_values, inst_values, zero4, zero4, theta, zero4, ct, n, 1)
        rows, total = E.lookup_missing_rows(ci, ct, usable, max_rows)
        if total:
            failures.append(WitnessFailure("lookup", li, rows, total))
    if cs.permutation:
        cols = [{"fixed": fixed, "advice": advice_values, "instance": inst_values}[kind][c] for kind, c in cs.permutation]
        for c, (total, cells) in enumerate(E.copy_mismatches(cols, pk.sigma_values, usable, max_rows)):
            if total:
                failures.append(WitnessFailure("copy", c, [r for r, _, _ in cells], total, [(c2, r2) for _, c2, r2 in cells]))
    return failures


# ---- proving-key check --------------------------------------------------------------------------------------------
class KeyFailure(namedtuple("KeyFailure", "kind index rows total")):
    """One failing part of a proving key (check_pk). kind and index:
      "fixed_commitment" / "sigma_commitment" (column): the VK point is not commit_lagrange of the column's values under the
        engine's params (rows None, total 1);
      "fixed_poly" / "sigma_poly" (column): the Lagrange rows where the NTT of the stored coefficients differs from the stored
        values;
      "fixed_coset" / "sigma_coset" (column), "l_coset" (0 l0, 1 l_last, 2 l_active): resident keys only, the extended rows
        where the stored coset differs from the coset NTT of the stored coefficients (of l_polys for the l cosets);
      "sigma_label" / "sigma_blinding" / "sigma_unlabelled" (permutation column): the three kinds of spb_sigma_check_dev, the
        rows i < u whose sigma labels no usable cell, the rows i >= u that are not fixed points, and the cells no sigma labels.
    rows: the first failing rows, ascending; total: how many rows fail."""


KEY_FAILURE_KINDS = ("fixed_commitment", "sigma_commitment", "fixed_poly", "sigma_poly", "fixed_coset", "sigma_coset", "l_coset", "sigma_label",
                     "sigma_blinding", "sigma_unlabelled")


def check_pk(E, pk, max_rows=16, timings=None):
    """Audit a proving key against the engine's params and against itself: a list of KeyFailure in the order of
    KEY_FAILURE_KINDS, ascending by index within a kind; [] for a sound key. Works on every residency mode; nothing is written
    to the key, and every temporary is freed before it returns.

    Values are the reference: a polynomial is compared as NTT(coefficients) against the values and a coset as the coset NTT of
    the coefficients against the stored coset, so one corrupted value or coset row is reported as that row. The commitments
    are recomputed from the values with one batch of nf + m MSMs, so a key made under other params shows as exactly nf + m
    commitment failures. The row comparisons go through one temporary of at most 2^extended_k rows (n rows for a lean key):
    recompute, subtract the stored buffer (vec_axpy with -1), report the nonzero rows. pk.vk_digest is not checked.
    timings: as create_proof's, a dict that gets the wall time of the stages commitments / polys / cosets / sigma."""
    import time
    t_last = [time.perf_counter()]

    def lap(name):
        if timings is not None:
            E.sync(); t = time.perf_counter(); timings[name] = timings.get(name, 0.0) + t - t_last[0]; t_last[0] = t
    n, ext = pk.n, 1 << E.extended_k
    minus_one = fr_mont(R_MOD - 1)
    nf, m = len(pk.fixed_values), len(pk.sigma_values)
    failures = []
    values = pk.fixed_values + pk.sigma_values
    got = E.commit(halo2.BASIS_G_LAGRANGE, values, n) if values else []
    for i, (want, have) in enumerate(zip(pk.fixed_commitments + pk.sigma_commitments, got)):
        if tuple(want) != tuple(have):
            failures.append(KeyFailure("fixed_commitment" if i < nf else "sigma_commitment", i if i < nf else i - nf, None, 1))
    lap("commitments")

    def compare(kind, index, tmp, stored, rows):
        E.vec_axpy(tmp, minus_one, stored, rows)
        bad, total = E.nonzero_rows(tmp, 0, rows, max_rows)
        if total:
            failures.append(KeyFailure(kind, index, bad, total))

    for kind, vals, coeffs in (("fixed_poly", pk.fixed_values, pk.fixed_polys), ("sigma_poly", pk.sigma_values, pk.sigma_polys)):
        for i, (v, p) in enumerate(zip(vals, coeffs)):
            tmp = E.clone(p)
            E.coeff_to_lagrange(tmp)
            compare(kind, i, tmp, v, n)
            del tmp
    lap("polys")
    if not pk.lean:
        for kind, coeffs, cosets in (("fixed_coset", pk.fixed_polys, pk.fixed_cosets), ("sigma_coset", pk.sigma_polys, pk.sigma_cosets)):
            for i, (p, c) in enumerate(zip(coeffs, cosets)):
                tmp = E.coeff_to_extended(p)
                compare(kind, i, tmp, c, ext)
                del tmp
        ls = l_polys(E, n, pk.usable_rows)
        for i, c in enumerate((pk.l0, pk.l_last, pk.l_active)):
            tmp = E.coeff_to_extended(ls[i])
            compare("l_coset", i, tmp, c, ext)
            del tmp
        del ls
        lap("cosets")
    if m:
        report = E.sigma_check(pk.sigma_values, pk.usable_rows, max_rows)
        for q, kind in enumerate(("sigma_label", "sigma_blinding", "sigma_unlabelled")):
            for c in range(m):
                total, rows = report[c][q]
                if total:
                    failures.append(KeyFailure(kind, c, rows, total))
        lap("sigma")
    return failures
