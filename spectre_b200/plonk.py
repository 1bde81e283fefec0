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
import os
import secrets
import time
from collections import namedtuple

import numpy as np

from . import halo2, poseidon
from .halo2 import FQ_MONT_INV, MONT_RADIX, P_MOD, R_MOD, g1_on_curve
from .transcript import EvmTranscriptRead, keccak256

_MONT = MONT_RADIX % R_MOD
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

# ---- curve points on the host: each Fq coordinate as its Montgomery limbs, 32 little-endian bytes; the G1 identity is
# (0, 0), a G2 point is ((x.c0, x.c1), (y.c0, y.c1)) -------------------------------------------------------------------------
_FQ_MONT = MONT_RADIX % P_MOD


def _fq_bytes(vals):
    return b"".join((v * _FQ_MONT % P_MOD).to_bytes(32, "little") for v in vals)


def _fq_int(raw):
    return int.from_bytes(raw, "little") * FQ_MONT_INV % P_MOD


def _limbs(raw):
    return np.frombuffer(raw, dtype="<u8").astype(np.uint64)


def _g1_from(raw):
    """(x, y) ints of a G1 point given as 64 bytes of limbs"""
    return _fq_int(raw[:32]), _fq_int(raw[32:64])


def _g1_limbs(pt):
    return _limbs(_fq_bytes(pt))


def _g2_limbs(q):
    """uint64[16] in the params trailer's order x.c0, x.c1, y.c0, y.c1"""
    return _limbs(_fq_bytes(v for c in q for v in c))


def _neg_g2(q):
    """-Q for a G2 point as uint64[16] limbs: x as given, both y coordinates negated mod p"""
    raw = np.asarray(q, dtype=np.uint64).reshape(16).tobytes()
    return _limbs(raw[:64] + _fq_bytes(-_fq_int(raw[i:i + 32]) % P_MOD for i in (64, 96)))


def write_pk(E, pk, path):
    """ProvingKey::write(writer, SerdeFormat::RawBytesUnchecked): header and commitments from the host, every polynomial
    streamed from device memory by the engine. A lean key writes the same bytes: each coset is rebuilt into one temporary
    buffer, appended and freed before the next."""
    with open(path, "wb") as f:
        f.write(pk.k.to_bytes(4, "big") + len(pk.fixed_commitments).to_bytes(4, "big"))
        for pt in pk.fixed_commitments + pk.sigma_commitments:
            f.write(_fq_bytes(pt))

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
    return None if g1_on_curve(*_g1_from(raw)) else "not on the curve"


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
    pts = [_g1_from(raw) for raw in raws]
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


def proof_evaluations(cs, n_sets, blinding_factors):
    """(evals, openings) for a proof of `cs` with n_sets permutation sets. evals: the evaluations a proof carries, each as
    (poly id, rotation), in transcript order: the advice queries, the fixed queries, the vanishing argument's random
    polynomial, sigma, per permutation set z, z(omega X) and, but for the last set, z(omega^-(bf+1) X), per lookup z,
    z(omega X), a', a'(omega^-1 X), s'. openings: create_proof's multi-open query order, which fixes SHPLONK's rotation sets,
    as positions in evals; position len(evals) is h at x, the one query the transcript does not carry.
    poly ids: ("advice", c), ("fixed", c), ("random",), ("sigma", c), ("perm", set), ("lk_z" | "lk_a" | "lk_s", lookup), ("h",)."""
    last = -(blinding_factors + 1)
    evals = [(("advice", c), r) for c, r in cs.advice_queries] + [(("fixed", c), r) for c, r in cs.fixed_queries]
    evals += [(("random",), 0)] + [(("sigma", c), 0) for c in range(len(cs.permutation))]
    for s in range(n_sets):
        evals += [(("perm", s), 0), (("perm", s), 1)] + ([(("perm", s), last)] if s + 1 < n_sets else [])
    for li in range(len(cs.lookups)):
        evals += [(("lk_z", li), 0), (("lk_z", li), 1), (("lk_a", li), 0), (("lk_a", li), -1), (("lk_s", li), 0)]
    at = {e: i for i, e in enumerate(evals)}
    kinds = lambda *ks: [i for i, ((kind, *_), _) in enumerate(evals) if kind in ks]
    openings = kinds("advice") + [at[(("perm", s), r)] for s in range(n_sets) for r in (0, 1)]
    openings += [at[(("perm", s), last)] for s in reversed(range(n_sets - 1))]
    openings += [at[e] for li in range(len(cs.lookups))
                 for e in ((("lk_z", li), 0), (("lk_a", li), 0), (("lk_s", li), 0), (("lk_a", li), -1), (("lk_z", li), 1))]
    return evals, openings + kinds("fixed", "sigma") + [len(evals), at[(("random",), 0)]]


def _by_poly_id(advice, fixed, sigma, perm, lookup_z, lookup_a, lookup_s, random, h):
    """{poly id of proof_evaluations: item}, the items of each kind given in column, set or lookup order"""
    out = {("random",): random, ("h",): h}
    for kind, items in (("advice", advice), ("fixed", fixed), ("sigma", sigma), ("perm", perm), ("lk_z", lookup_z), ("lk_a", lookup_a),
                        ("lk_s", lookup_s)):
        out.update(((kind, i), v) for i, v in enumerate(items))
    return out


def _intake(who, cs, n, usable, instances, advice_columns=None, E=None):
    """Refuse instance and advice columns the circuit cannot take, as upstream does (`who` prefixes the message); advice is
    checked when given. With an engine, the instance columns uploaded as create_proof lays them out: each column's values
    at rows 0..len of an n-row buffer, zero below."""
    if len(instances) != cs.num_instance:
        raise ValueError("%s: %d instance columns given, the circuit has %d (upstream: Error::InvalidInstances)" % (who, len(instances), cs.num_instance))
    if advice_columns is not None and len(advice_columns) != cs.num_advice:
        raise ValueError("%s: %d advice columns given, the circuit has %d" % (who, len(advice_columns), cs.num_advice))
    for col in instances:
        if len(col) > usable:
            raise ValueError("%s: an instance column has more than %d values (upstream: Error::InstanceTooLarge)" % (who, usable))
    if E is None:
        return None
    values = []
    for col in instances:
        b = E.alloc(n); E.write_rows(b, 0, fr_mont_rows(col)); values.append(b)
    return values


def _permutation_columns(cs, fixed, advice, instance):
    """the column behind each cs.permutation entry (kind, c): fixed[c], advice[c] or instance[c], whatever the containers hold"""
    by_kind = {"fixed": fixed, "advice": advice, "instance": instance}
    return [by_kind[kind][c] for kind, c in cs.permutation]


def _compressed_lookup(E, pk, li, theta, advice_values, inst_values):
    """lookup li's input and table expressions, each compressed with theta (a Horner sum over the tuple) into an n-row buffer"""
    cs, n, zero4 = pk.cs, pk.n, fr_mont(0)
    ci, ct = E.alloc(n), E.alloc(n)
    for exprs, out in zip(cs.lookups[li], (ci, ct)):
        E.graph_evaluate(cs.lookup_compress_program(exprs), pk.fixed_values, advice_values, inst_values, zero4, zero4, theta, zero4, out, n, 1)
    return ci, ct


def _stage_timer(E, timings):
    """lap(name): with a timings dict, sync the engine and add the wall time since the previous lap (or since this call) to
    timings[name]; without one, nothing"""
    t_last = [time.perf_counter()]

    def lap(name):
        if timings is not None:
            E.sync(); t = time.perf_counter(); timings[name] = timings.get(name, 0.0) + t - t_last[0]; t_last[0] = t
    return lap


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
    cols = _permutation_columns(cs, fixed_p, advice_p, inst_p)
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
    cs, k, n = pk.cs, pk.k, pk.n
    bf, usable = pk.blinding_factors, pk.usable_rows
    ext_n, rot_scale = 1 << E.extended_k, 1 << (E.extended_k - k)
    G, GL = halo2.BASIS_G, halo2.BASIS_G_LAGRANGE
    w = omega_of(k)
    lap = _stage_timer(E, timings)

    # 1. vk, instances
    inst_values = _intake("create_proof", cs, n, usable, instances, advice_columns, E)
    for col in instances:
        for v in col:
            transcript.common_scalar(v)                      # KZG: instances enter the transcript, no commitments
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
    for li in range(len(cs.lookups)):
        L = _L()
        L.compressed_input, L.compressed_table = _compressed_lookup(E, pk, li, theta, advice_values, inst_values)
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
    col_values = _permutation_columns(cs, pk.fixed_values, advice_values, inst_values)
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
            cosets = _permutation_columns(cs, fixed_cosets, advice_cosets, inst_cosets)
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
    x_pow = lambda rot: x * pow(w, rot % n, R_MOD) % R_MOD

    # 8. evaluations: every (polynomial, point) query, h last, is evaluated by ONE engine call (one kernel launch for the whole
    # list), then the scalars but h's enter the transcript in the order the verifier reads them.
    # vanishing::evaluate: h(X) = sum_i x^(n i) h_i(X), and the random polynomial at x
    h_poly = E.alloc(n)
    E.lincomb(h_pieces, fr_mont(pow(x, n, R_MOD)), h_poly, n)
    polys = _by_poly_id(advice_polys, pk.fixed_polys, pk.sigma_polys, perm_polys, [L.product_poly for L in lookups],
                        [L.permuted_input_poly for L in lookups], [L.permuted_table_poly for L in lookups], random_poly, h_poly)
    evals, openings = proof_evaluations(cs, len(perm_polys), bf)
    asked = [(pid, x_pow(rot)) for pid, rot in evals + [(("h",), 0)]]
    values = eval_polynomial_many(E, [(polys[pid], pt) for pid, pt in asked], n)
    for e in values[:-1]:
        transcript.write_scalar(e)
    lap("evaluations")

    # 9. multi-open queries in create_proof's order
    evals_q = [asked[i] + (values[i],) for i in openings]
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
    inst_values = _intake("check_witness", cs, n, usable, instances, advice_columns, E)
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
    for li in range(len(cs.lookups)):
        ci, ct = _compressed_lookup(E, pk, li, theta, advice_values, inst_values)
        rows, total = E.lookup_missing_rows(ci, ct, usable, max_rows)
        if total:
            failures.append(WitnessFailure("lookup", li, rows, total))
    if cs.permutation:
        cols = _permutation_columns(cs, fixed, advice_values, inst_values)
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
    lap = _stage_timer(E, timings)
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


# ---- params check -------------------------------------------------------------------------------------------------
class ParamsFailure(namedtuple("ParamsFailure", "kind index detail")):
    """One failing part of a ParamsKZG (check_params). kind and index:
      "g_generator" (0): g[0] is not the G1 generator (1, 2), or is not vp.g;
      "g2_generator" (0): vp.g2 is not halo2curves' G2 generator;
      "trailer" (0 g2, 1 s_g2): the handle's own G2 trailer differs from the vp given;
      "s_g2" (0): the pairing refuses vp.s_g2 (off the curve or outside the G2 subgroup), detail = the library's error text;
      "powers" (j): the smallest j >= 1 with g[j] != s g[j - 1] for the s of vp.s_g2;
      "lagrange" (i): the smallest i with g_lagrange[i] != g_to_lagrange(g)[i], g as stored.
    detail: a human-readable reason."""


PARAMS_FAILURE_KINDS = ("g_generator", "g2_generator", "trailer", "s_g2", "powers", "lagrange")

# halo2curves' G2Affine::generator (EIP-197): ((x.c0, x.c1), (y.c0, y.c1))
G2_GENERATOR = ((0x1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed, 0x198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2),
                (0x12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa, 0x090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b))


def check_params(E, be, vp=None, seed=None, timings=None):
    """Check that the points of the engine's params fit together: a list of ParamsFailure in the order of PARAMS_FAILURE_KINDS,
    [] for sound params. E: an engine bound to the params (E.params, E.k == params.k); be: anything with pairing_check_batch(ps,
    qs, m) in halo2.Backend's layouts, whose refusal of an input raises halo2.BackendError; vp: the halo2.ParamsVerifierKZG the
    proofs will be verified against (a verifier contract's constants, say), by default params.verifier_params(); seed: 32 bytes
    for the ChaCha20 draws (default os.urandom(32)), the same seed giving the same report. A handle without a 2^k SRS and its
    g_lagrange (from_bases) raises ValueError. Nothing is written to the params, and every temporary is freed before it returns.

    Every n-row vector stays on the engine: the draws, their inverse NTT and the MSMs, which go through the window tables of a
    handle that has them. Only points and verdicts reach the host.
      * powers: with r drawn at random, A = sum_{i<m} r_i g[i] and B = sum_{i<m} r_i g[i+1] (two prefix MSMs over one draw). The
        chain g[j] = s g[j-1] holds for every j <= m exactly when B = s A, decided by one pairing check e(B, g2) e(A, -s_g2) = 1.
        m = n - 1 first; if it fails, a bisection over m with fresh draws per step (ceil(log2 n) more checks) finds the first j.
        When the pairing refuses vp.s_g2 (reported as s_g2) or vp.g2 (reported as g2_generator), powers is not checked.
      * lagrange: with v drawn at random and c = lagrange_to_coeff(v), MSM(v, g_lagrange) = MSM(c, g) holds exactly when
        g_lagrange = g_to_lagrange(g) (the basis downsize computes from g). No pairing. If it fails, a bisection with v zeroed
        past m, one inverse NTT and one full MSM over g per step, finds the first row.
    Soundness: G1 has prime order r, so a wrong prefix passes one check with probability at most 1/r over the draws. The checks
    are random linear combinations: they cannot count failures, so each kind reports its first failure only.
    timings: a dict that gets the wall time of the stages points / powers / lagrange."""
    params = E.params
    if E.k != params.k:
        raise ValueError("check_params: the engine is for k = %d, the params for k = %d" % (E.k, params.k))
    n = 1 << params.k
    G, GL = halo2.BASIS_G, halo2.BASIS_G_LAGRANGE
    refused = "check_params: the handle holds no 2^k SRS with its g_lagrange (from_bases bases are not params)"
    if params.n != n:
        raise ValueError(refused)
    try:
        params.get_g(0, 1, basis=GL)
    except halo2.BackendError:
        raise ValueError(refused) from None
    g0 = params.get_g(0, 1)[0]
    own_g2, own_s_g2 = params.get_g2()
    has_trailer = own_g2.any() and own_s_g2.any()
    given = vp is not None
    vp = params.verifier_params() if vp is None else vp
    seed = os.urandom(32) if seed is None else seed
    lap = _stage_timer(E, timings)
    drawn = [0]

    def draw(rows):
        """fresh draws: each call takes the next `rows` elements of the seed's stream"""
        drawn[0] += rows
        return E.random_chacha(seed, drawn[0] - rows, rows)

    # ---- points: the generators and the trailer, on the host --------------------------------------------------------
    failures = []
    generator = _g1_limbs((1, 2))
    if not np.array_equal(g0, generator) or not np.array_equal(g0, vp.g):
        failures.append(ParamsFailure("g_generator", 0, "g[0] is %s, the G1 generator is (1, 2) and vp.g is %s"
                                      % (_g1_from(g0.tobytes()), _g1_from(vp.g.tobytes()))))
    g2_ok = np.array_equal(vp.g2, _g2_limbs(G2_GENERATOR))
    if not g2_ok:
        failures.append(ParamsFailure("g2_generator", 0, "vp.g2 is not the G2 generator"))
    if given and has_trailer:
        for i, (own, want) in enumerate(((own_g2, vp.g2), (own_s_g2, vp.s_g2))):
            if not np.array_equal(own, want):
                failures.append(ParamsFailure("trailer", i, "the params' own %s differs from vp's" % ("g2", "s_g2")[i]))
                break
    lap("points")

    # ---- powers: g[j] = s g[j-1] -----------------------------------------------------------------------------------
    neg_s_g2 = _neg_g2(vp.s_g2)

    def chain_holds(m):
        """g[j] = s g[j-1] for 1 <= j <= m: d = (0, r_0 .. r_{m-1}, 0), A = MSM(d[1:m+2]) and B = MSM(d[0:m+1]) over g[0..m]"""
        d = draw(m + 2)
        E.zero(E.view(d, 0, 1)); E.zero(E.view(d, m + 1, m + 2))
        a, b = E.commit(G, [E.view(d, 1, m + 2), E.view(d, 0, m + 1)], m + 1)
        del d
        return be.pairing_check_batch(np.stack([_g1_limbs(b), _g1_limbs(a)]), np.stack([vp.g2, neg_s_g2]), 2)[0]
    if n > 1:
        try:
            whole = chain_holds(n - 1)
        except halo2.BackendError as error:                 # a trailer point refused: find out whether it is s_g2
            whole = None
            try:
                be.pairing_check_batch(np.zeros((1, 8), dtype=np.uint64), vp.s_g2.reshape(1, 16), 1)
            except halo2.BackendError as e:
                failures.append(ParamsFailure("s_g2", 0, str(e)))
            else:
                if g2_ok:                                   # the generator and s_g2 both pass: not a verdict on the points
                    raise error
                # else vp.g2 was refused, and g2_generator already names it
        if whole is False:
            lo, hi = 0, n - 1                               # the chain holds up to lo and breaks by hi
            while hi - lo > 1:
                mid = (lo + hi) // 2
                if chain_holds(mid):
                    lo = mid
                else:
                    hi = mid
            failures.append(ParamsFailure("powers", hi, "g[%d] is not s g[%d]" % (hi, hi - 1)))
    lap("powers")

    # ---- lagrange: g_lagrange = g_to_lagrange(g) -------------------------------------------------------------------
    def rows_hold(m):
        """g_lagrange[i] = g_to_lagrange(g)[i] for i < m: v zeroed past m, MSM(v, g_lagrange) = MSM(lagrange_to_coeff(v), g)"""
        v = draw(n)
        if m < n:
            E.zero(E.view(v, m, n))
        c = E.clone(v)
        E.lagrange_to_coeff(c)
        lhs = E.commit(GL, [v], m)[0]
        del v
        rhs = E.commit(G, [c], n)[0]
        return tuple(lhs) == tuple(rhs)
    if not rows_hold(n):
        lo, hi = 0, n                                       # rows < lo agree, some row < hi does not
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if rows_hold(mid):
                lo = mid
            else:
                hi = mid
        failures.append(ParamsFailure("lagrange", hi - 1, "g_lagrange[%d] is not row %d of g_to_lagrange(g)" % (hi - 1, hi - 1)))
    lap("lagrange")
    return failures


# ---- multi-party params: a powers-of-tau update chain ---------------------------------------------------------------
# Each party i draws t_i, maps g[j] -> t_i^j g[j] and [s]_2 -> t_i [s]_2 (ParamsKZG.contribute) and publishes a ParamsUpdate.
# If any one party erased its t_i, nobody knows the final secret s_0 t_1 ... t_m, whoever made the starting params.
PARAMS_UPDATE_DOMAIN = b"spectre-b200 params update v1"
PARAMS_UPDATE_BYTES = 128 + 64 + 64 + 32


class ParamsUpdate(namedtuple("ParamsUpdate", "s_g2 t_g1 r_g1 z")):
    """The public record of one powers-of-tau update: s_g2 = [s]_2 after the update (uint64[16], the params trailer's layout),
    t_g1 = T = t G1 and r_g1 = R = rho G1 (uint64[8] each, G1 affine limbs) and z = rho + c t mod r (an int), a Schnorr proof
    that the party knew t, with c = params_update_challenge(the [s]_2 before, this record).

    to_bytes / from_bytes: s_g2 (128 B) | T (64 B) | R (64 B) | z (32 B). Every coordinate is its Montgomery limbs as the params
    file's trailer stores them, and z is its Fr Montgomery limbs, all little-endian."""

    def to_bytes(self):
        return b"".join(np.ascontiguousarray(a, dtype="<u8").tobytes() for a in (self.s_g2, self.t_g1, self.r_g1, fr_mont(self.z)))

    @classmethod
    def from_bytes(cls, data):
        """The inverse of to_bytes. ValueError for a wrong length, a coordinate or z not canonical, or a G1 point off the curve
        (the G2 point's curve and subgroup are checked where the pairing takes it)."""
        data = bytes(data)
        if len(data) != PARAMS_UPDATE_BYTES:
            raise ValueError("ParamsUpdate.from_bytes: %d bytes, the record is %d" % (len(data), PARAMS_UPDATE_BYTES))
        if any(int.from_bytes(data[i:i + 32], "little") >= P_MOD for i in range(0, 128, 32)):
            raise ValueError("ParamsUpdate.from_bytes: s_g2: a coordinate is not less than the field modulus")
        for name, raw in (("T", data[128:192]), ("R", data[192:256])):
            why = _point_check(raw)
            if why:
                raise ValueError("ParamsUpdate.from_bytes: %s: %s" % (name, why))
        if int.from_bytes(data[256:], "little") >= R_MOD:
            raise ValueError("ParamsUpdate.from_bytes: z is not less than r")
        return cls(_limbs(data[:128]), _limbs(data[128:192]), _limbs(data[192:256]), fr_int(_limbs(data[256:])))


def params_update_challenge(s_g2_before, update):
    """c = keccak256(b"spectre-b200 params update v1" || s_g2 before || s_g2 after || T || R), read big-endian, mod r, each point
    in the bytes of ParamsUpdate.to_bytes. This is this project's own encoding, not an external standard: a record is checked
    only by this code. Binding the [s]_2 before makes a record valid at its own place in the chain only."""
    data = PARAMS_UPDATE_DOMAIN + b"".join(np.ascontiguousarray(a, dtype="<u8").tobytes() for a in (s_g2_before, update.s_g2, update.t_g1, update.r_g1))
    return int.from_bytes(keccak256(data), "big") % R_MOD


def prove_params_update(be, s_g2_before, s_g2_after, t, rho):
    """The ParamsUpdate of the update by t from s_g2_before to s_g2_after, with the Schnorr nonce rho (ints in [1, r)). be:
    anything with best_multiexp(coeffs, bases) in halo2.Backend's layouts."""
    t_g1, r_g1 = (_g1_limbs(_multiexp(be, [v], [(1, 2)])) for v in (t, rho))
    update = ParamsUpdate(np.asarray(s_g2_after, dtype=np.uint64).reshape(16).copy(), t_g1, r_g1, 0)
    return update._replace(z=(rho + params_update_challenge(s_g2_before, update) * t) % R_MOD)


def _random_fr():
    """Fr::random's rule: 64 bytes of os.urandom read little-endian, reduced mod r (from_u512)"""
    return int.from_bytes(os.urandom(64), "little") % R_MOD


def contribute_params(be, params, secret=None, nonce=None):
    """One party's powers-of-tau update of params (a halo2.ParamsKZG with its G2 trailer and no window tables): returns
    (new params, ParamsUpdate). secret = t and nonce = rho, ints in [1, r), are drawn as Fr::random draws them when None. The
    input params stay valid and unchanged.

    The party must erase t (and rho) afterwards: anyone who learns every party's t can forge proofs. Python cannot scrub
    memory (ints are immutable and may be copied), so a caller who needs erasure runs the contribution in a process that exits
    once it has written the new params file and the record."""
    t = _random_fr() if secret is None else secret
    rho = _random_fr() if nonce is None else nonce
    if not 0 < t < R_MOD or not 0 < rho < R_MOD:
        raise ValueError("contribute_params: the secret and the nonce must lie in [1, r)")
    s_before = params.get_g2()[1]
    new = params.contribute(fr_mont(t))
    return new, prove_params_update(be, s_before, new.get_g2()[1], t, rho)


class UpdateFailure(namedtuple("UpdateFailure", "kind index detail")):
    """One failing record of a params update chain (check_params_updates), index = its place in the chain. At most one per record,
    the first of:
      "degenerate": T or the record's s_g2 is the identity;
      "ratio": e(T, s_before) != e(G1, s_g2): the record's [s]_2 is not t times the one before it (a record out of place, a T
        for another t, or an s_g2 that does not follow);
      "knowledge": z G1 != R + c T, so the record does not prove that its party knew t.
    detail: a human-readable reason."""


def check_params_updates(E, be, start_vp, updates, seed=None):
    """Check a powers-of-tau update chain and the params it ends in: a list of UpdateFailure in chain order, then the ParamsFailure
    list of check_params against [s]_2 of the last record; [] for a sound chain. E: an engine bound to the final params; be:
    anything with best_multiexp and pairing_check_batch in halo2.Backend's layouts; start_vp: the ParamsVerifierKZG of the params
    the chain starts from (s_0 = start_vp.s_g2); updates: the ParamsUpdate records in order; seed: check_params' seed.

    Per record, one 3-term best_multiexp decides knowledge (z G1 - c T - R = O). Every ratio check e(T_i, s_{i-1}) e(-G1, s_i) = 1
    goes into one pairing_check_batch call of len(updates) checks of two pairs. Then check_params(E, be, ParamsVerifierKZG(G1,
    start_vp.g2, s_m)) shows that the final params are the powers of that s_m."""
    generator, neg_generator = _g1_limbs((1, 2)), _g1_limbs((1, P_MOD - 2))
    prev = np.asarray(start_vp.s_g2, dtype=np.uint64).reshape(16)
    ps, qs, found = [], [], []
    for i, u in enumerate(updates):
        s_after = np.asarray(u.s_g2, dtype=np.uint64).reshape(16)
        if not np.asarray(u.t_g1).any() or not s_after.any():
            found.append(UpdateFailure("degenerate", i, "T is the identity" if not np.asarray(u.t_g1).any() else "s_g2 is the identity"))
        else:
            c = params_update_challenge(prev, u)
            rest = halo2.jacobian_to_affine_ints(be.best_multiexp(fr_mont_rows([u.z, R_MOD - c, R_MOD - 1]), np.stack([generator, u.t_g1, u.r_g1])))
            found.append(None if rest == (0, 0) else UpdateFailure("knowledge", i, "z G1 is not R + c T"))
        ps += [u.t_g1, neg_generator]
        qs += [prev, s_after]
        prev = s_after
    if updates:
        ok = be.pairing_check_batch(np.stack(ps), np.stack(qs), 2)
        for i, holds in enumerate(ok):
            if not holds and (found[i] is None or found[i].kind != "degenerate"):
                found[i] = UpdateFailure("ratio", i, "s_g2 of record %d is not t s_g2 of the one before it" % i)
    failures = [f for f in found if f is not None]
    return failures + check_params(E, be, halo2.ParamsVerifierKZG(generator, start_vp.g2, prev), seed=seed)


# ---- verifier -----------------------------------------------------------------------------------------------------
# [UPSTREAM] halo2_proofs/src/plonk/verifier.rs verify_proof with VerifierSHPLONK and SingleStrategy
# (poly/kzg/multiopen/shplonk/verifier.rs, poly/kzg/strategy.rs): what snark_verifier_sdk::gen_proof runs on every proof it
# makes. The transcript replay and the quotient identity are host work on a few hundred bytes; the device does the one
# multiexp per proof (a few dozen terms) and the pairing check, so a batch of proofs is decided by one pairing launch sequence.
class VerifyingKey(namedtuple("VerifyingKey", "cs k vk_digest fixed_commitments sigma_commitments")):
    """The part of a proving key a verifier reads: the constraint system, k, the transcript digest and the commitments to the
    fixed and permutation (sigma) columns, as affine (x, y) ints."""


def verifying_key(pk):
    return VerifyingKey(pk.cs, pk.k, pk.vk_digest, list(pk.fixed_commitments), list(pk.sigma_commitments))


class ProofFailure(namedtuple("ProofFailure", "kind detail")):
    """Why verify_proof rejects a proof. kind "transcript": the proof bytes cannot be read (too short, trailing bytes, a scalar
    >= r, a point off the curve, or anything else the reading transcript refuses); "opening": the bytes read, but the SHPLONK
    opening's pairing check fails. With accumulator indices (an aggregation proof, checked as its verifier contract does) two
    more: "accumulator_encoding": the 12 instance limbs of the KZG accumulator do not decode to two curve points
    (accumulator_from_limbs), decided on the host; "accumulator": they decode, but e(lhs, [1]_2) e(rhs, -[s]_2) != 1, so the
    inner snark the accumulator stands for is invalid. The first failure in the order transcript, accumulator_encoding,
    opening, accumulator is reported. detail: a human-readable reason."""


def _multiexp(be, scalars, points):
    """sum_i scalars[i] points[i] on the backend, for ints and affine int points; the identity is (0, 0)"""
    return halo2.jacobian_to_affine_ints(be.best_multiexp(fr_mont_rows(scalars), np.stack([_g1_limbs(c) for c in points])))


def _opening_points(be, vp, vk, instances, proof, transcript_read):
    """Replay one proof up to the SHPLONK verifier's two G1 points (P1, P2), the opening holding iff
    e(P1, [1]_2) e(P2, -[s]_2) = 1; a ProofFailure("transcript", ...) when the bytes cannot be read."""
    got = _opening_terms(vp, vk, instances, proof, transcript_read)
    if isinstance(got, ProofFailure):
        return got
    scalars, bases, h2 = got
    return _multiexp(be, scalars, bases), h2


def _opening_terms(vp, vk, instances, proof, transcript_read):
    """The host part of _opening_points: (scalars, bases, P2) with P1 = sum_i scalars[i] bases[i], or the ProofFailure"""
    cs, k = vk.cs, vk.k
    n = 1 << k
    bf = cs.blinding_factors()
    usable = n - (bf + 1)
    _intake("verify_proof", cs, n, usable, instances)
    if len(vk.fixed_commitments) != cs.num_fixed or len(vk.sigma_commitments) != len(cs.permutation):
        raise ValueError("verify_proof: the verifying key has %d fixed and %d sigma commitments, the circuit %d and %d"
                         % (len(vk.fixed_commitments), len(vk.sigma_commitments), cs.num_fixed, len(cs.permutation)))
    w = omega_of(k)
    R = R_MOD
    try:
        T = transcript_read(vk.vk_digest, bytes(proof))

        def rd(f):
            v = f()
            if T.pos > len(T.stream):
                raise ValueError("the proof ends early (%d bytes)" % len(T.stream))
            return v
        pt, sc = lambda: rd(T.read_ec_point), lambda: rd(T.read_scalar)
        for col in instances:
            for v in col:
                T.common_scalar(v)
        advice_c = [pt() for _ in range(cs.num_advice)]
        theta = T.squeeze_challenge()
        permuted_c = [(pt(), pt()) for _ in cs.lookups]
        beta = T.squeeze_challenge(); gamma = T.squeeze_challenge()
        chunk = max(1, cs.chunk_len())
        n_sets = -(-len(cs.permutation) // chunk) if cs.permutation else 0
        perm_c = [pt() for _ in range(n_sets)]
        lookz_c = [pt() for _ in cs.lookups]
        random_c = pt()
        y = T.squeeze_challenge()
        h_c = [pt() for _ in range(cs.degree() - 1)]
        x = T.squeeze_challenge()
        evals, openings = proof_evaluations(cs, n_sets, bf)
        got = dict(zip(evals, [sc() for _ in evals]))                  # (poly id, rotation) -> the proof's evaluation
        y2 = T.squeeze_challenge(); v = T.squeeze_challenge()
        h1 = pt()
        u = T.squeeze_challenge()
        h2 = pt()
        if T.pos != len(T.stream):
            return ProofFailure("transcript", "%d trailing bytes after the proof" % (len(T.stream) - T.pos))
    except ValueError as e:
        return ProofFailure("transcript", str(e))

    # ---- the quotient identity at x: the h(x) the proof must open to --------------------------------------------------
    xn = pow(x, n, R)
    inv = lambda a: pow(a % R, -1, R)
    inst_rots = sorted({r for _, r in cs.instance_queries})
    max_inst = max([len(c) for c in instances] or [0])
    rows = set([0, usable] + list(range(usable + 1, n)) + [i - r for r in inst_rots for i in range(max_inst)])
    L = {i: (xn - 1) * pow(w, i % n, R) % R * inv(n * (x - pow(w, i % n, R))) % R for i in rows}
    l0, l_last = L[0], L[usable]
    l_active = (1 - l_last - sum(L[i] for i in range(usable + 1, n))) % R
    inst = {(c, r): sum(val * L[i - r] for i, val in enumerate(instances[c])) % R for c, r in cs.instance_queries}
    perm = lambda s, rot: got[(("perm", s), rot)]
    look = lambda kind, li, rot: got[((kind, li), rot)]

    def ev(e):
        t = e[0]
        if t == "const": return e[1]
        if t in ("fixed", "advice"): return got[((t, e[1]), e[2])]
        if t == "instance": return inst[(e[1], e[2])]
        if t == "neg": return -ev(e[1]) % R
        if t == "sum": return (ev(e[1]) + ev(e[2])) % R
        if t == "prod": return ev(e[1]) * ev(e[2]) % R
        if t == "scaled": return ev(e[1]) * e[2] % R
        raise ValueError("unknown expression node %r" % (t,))
    acc = 0
    for g in cs.gates:
        acc = (acc * y + ev(g)) % R
    if n_sets:
        cur = lambda kind, qs: {c: got[((kind, c), 0)] for c, r in qs if r == 0}
        cols = _permutation_columns(cs, cur("fixed", cs.fixed_queries), cur("advice", cs.advice_queries),
                                    {c: v for (c, r), v in inst.items() if r == 0})
        acc = (acc * y + l0 * (1 - perm(0, 0))) % R
        zl = perm(n_sets - 1, 0)
        acc = (acc * y + l_last * (zl * zl - zl)) % R
        for s in range(1, n_sets):
            acc = (acc * y + l0 * (perm(s, 0) - perm(s - 1, -(bf + 1)))) % R
        for s in range(n_sets):
            left, right = perm(s, 1), perm(s, 0)
            for c in range(s * chunk, min((s + 1) * chunk, len(cs.permutation))):
                left = left * (cols[c] + beta * got[(("sigma", c), 0)] + gamma) % R
                right = right * (cols[c] + beta * x % R * pow(DELTA, c, R) + gamma) % R
            acc = (acc * y + l_active * (left - right)) % R
    for li, (ins, tbs) in enumerate(cs.lookups):
        z, z_next, a_p, a_inv, s_p = look("lk_z", li, 0), look("lk_z", li, 1), look("lk_a", li, 0), look("lk_a", li, -1), look("lk_s", li, 0)
        ci = ct = 0
        for e in ins: ci = (ci * theta + ev(e)) % R
        for e in tbs: ct = (ct * theta + ev(e)) % R
        acc = (acc * y + l0 * (1 - z)) % R
        acc = (acc * y + l_last * (z * z - z)) % R
        acc = (acc * y + l_active * (z_next * (a_p + beta) % R * (s_p + gamma) - z * (ci + beta) % R * (ct + gamma))) % R
        acc = (acc * y + l0 * (a_p - s_p)) % R
        acc = (acc * y + l_active * (a_p - s_p) % R * (a_p - a_inv)) % R
    expected_h = acc * inv(xn - 1) % R

    # ---- SHPLONK: the queries in create_proof's order, one linear combination of commitments per opening ------------
    xw = lambda r: x * pow(w, r % n, R) % R
    # per polynomial, [(scalar, point)] summing to its commitment; h(X) = sum_i X^(n i) h_i(X)
    one = lambda pts: [[(1, p)] for p in pts]
    commits = _by_poly_id(one(advice_c), one(vk.fixed_commitments), one(vk.sigma_commitments), one(perm_c), one(lookz_c),
                          one(a for a, _ in permuted_c), one(s for _, s in permuted_c), [(1, random_c)],
                          [(pow(xn, i, R), hc) for i, hc in enumerate(h_c)])
    asked = [(pid, xw(rot), got[(pid, rot)]) for pid, rot in evals] + [(("h",), x, expected_h)]
    sets = rotation_sets([asked[i] for i in openings])
    super_pts = []
    for pts, _, _ in sets:
        for p in pts:
            if p not in super_pts: super_pts.append(p)

    def interp_eval(pts, evs, at):                            # the interpolation of (pts, evs) evaluated at `at`
        tot = 0
        for j, (pj, ej) in enumerate(zip(pts, evs)):
            num = den = 1
            for m, pm in enumerate(pts):
                if m != j:
                    num = num * (at - pm) % R; den = den * (pj - pm) % R
            tot = (tot + ej * num % R * inv(den)) % R
        return tot
    # P1 = (sum_ij v^i Z_{T\S_i}(u) y^j (C_ij - r_ij(u) G) - Z_T(u) h1) / Z_{T\S_0}(u) + u h2, P2 = h2:
    # the opening holds iff P1 = s h2, i.e. e(P1, [1]_2) e(P2, -[s]_2) = 1
    terms, const, z0 = {}, 0, None
    for i, (pts, pids, evs) in enumerate(sets):
        zi = 1
        for p in super_pts:
            if p not in pts: zi = zi * (u - p) % R
        if i == 0: z0 = zi
        outer = pow(v, i, R) * zi % R
        for j, pid in enumerate(pids):
            wij = outer * pow(y2, j, R) % R
            for s_, c in commits[pid]:
                terms[c] = (terms.get(c, 0) + wij * s_) % R
            const = (const + wij * interp_eval(pts, evs[j], u)) % R
    zt = 1
    for p in super_pts: zt = zt * (u - p) % R
    z0_inv = inv(z0)
    g = _g1_from(vp.g.tobytes())
    terms[g] = (terms.get(g, 0) - const) % R
    terms[h1] = (terms.get(h1, 0) - zt) % R
    bases = [c for c in terms]
    scalars = [terms[c] * z0_inv % R for c in bases]
    bases.append(h2); scalars.append(u)
    return scalars, bases, h2


# ---- the KZG accumulator of an aggregation proof ----------------------------------------------------------------------
# [UPSTREAM] snark-verifier's KzgAccumulator and KzgAs (pcs/kzg/accumulation.rs), and what the verifier contract its EVM
# loader generates does with the accumulator (contracts/snark-verifiers/sync_step_verifier.sol:213-236 decodes it,
# :1165-1208 folds it into the final pairing; committee_update_verifier.sol:214-237 and :1178-1221 alike). An aggregation
# circuit verifies its inner snark up to the pairing and exposes what is left, a pair (lhs, rhs) with the inner snark valid
# iff e(lhs, [1]_2) = e(rhs, [s]_2), as 12 public instances; that pairing is the outer proof's verifier's job.
class KzgAccumulator(namedtuple("KzgAccumulator", "lhs rhs")):
    """A KZG accumulator: two affine G1 points as (x, y) ints, valid iff e(lhs, [1]_2) e(rhs, -[s]_2) = 1."""


ACCUMULATOR_LIMBS, ACCUMULATOR_LIMB_BITS = 3, 88
# (column, row) of the 12 accumulator limbs among the instances, as snark-verifier's accumulator_indices: Spectre's
# aggregation circuits put them first in their one instance column
AGGREGATION_ACCUMULATOR_INDICES = [(0, i) for i in range(4 * ACCUMULATOR_LIMBS)]
_M256 = MONT_RADIX - 1                                  # an EVM word wraps mod 2^256


def accumulator_to_limbs(acc):
    """The 12 instance words of a KzgAccumulator: lhs.x, lhs.y, rhs.x, rhs.y, each as three 88-bit limbs, least significant first."""
    mask = (1 << ACCUMULATOR_LIMB_BITS) - 1
    return [(v >> (ACCUMULATOR_LIMB_BITS * i)) & mask for v in (acc.lhs[0], acc.lhs[1], acc.rhs[0], acc.rhs[1])
            for i in range(ACCUMULATOR_LIMBS)]


def accumulator_from_limbs(words):
    """The KzgAccumulator that 12 instance words encode, decoded exactly as the generated verifier contract decodes it, or None
    where the contract refuses it. Each word is first reduced mod r (the contract reads every instance as mod(calldataload, f_q));
    a coordinate is l0 + l1 2^88 + l2 2^176 with the EVM's wrap-around mod 2^256, so limbs of 88 bits or more overlap and are
    not refused; each point must pass validate_ec_point: x < p, y < p and y^2 = x^3 + 3, which refuses the identity (0, 0)."""
    words = [int(w) % R_MOD for w in words]
    if len(words) != 4 * ACCUMULATOR_LIMBS:
        raise ValueError("accumulator_from_limbs: %d words, an accumulator has %d" % (len(words), 4 * ACCUMULATOR_LIMBS))
    coords = []
    for c in range(4):
        v = 0
        for i, limb in enumerate(words[ACCUMULATOR_LIMBS * c:ACCUMULATOR_LIMBS * (c + 1)]):
            v = (v + (limb << (ACCUMULATOR_LIMB_BITS * i))) & _M256
        coords.append(v)
    pts = [(coords[0], coords[1]), (coords[2], coords[3])]
    if not all(g1_on_curve(x, y) for x, y in pts):
        return None
    return KzgAccumulator(*pts)


def _accumulator_words(instances, indices):
    indices = list(indices)
    if len(indices) != 4 * ACCUMULATOR_LIMBS:
        raise ValueError("accumulator_indices: %d given, an accumulator has %d limbs" % (len(indices), 4 * ACCUMULATOR_LIMBS))
    words = []
    for col, row in indices:
        if not (0 <= col < len(instances) and 0 <= row < len(instances[col])):
            raise ValueError("accumulator_indices: (%d, %d) is outside the instances" % (col, row))
        words.append(instances[col][row])
    return words


def _replay(be, vp, vk, instances, proof, transcript_read, indices):
    """(P1, P2, the decoded accumulator or None without indices), or the first ProofFailure: transcript, then
    accumulator_encoding, both found on the host before the one multiexp"""
    words = None if indices is None else _accumulator_words(instances, indices)
    got = _opening_terms(vp, vk, instances, proof, transcript_read)
    if isinstance(got, ProofFailure):
        return got
    acc = None
    if words is not None:
        acc = accumulator_from_limbs(words)
        if acc is None:
            return ProofFailure("accumulator_encoding", "the accumulator limbs in the instances are not two points on the curve")
    scalars, bases, h2 = got
    return _multiexp(be, scalars, bases), h2, acc


def succinct_verify(be, vp, vk, instances, proof, transcript_read=EvmTranscriptRead):
    """The accumulator a proof leaves for its aggregation: verify_proof without the final pairing (snark-verifier's succinct
    SHPLONK verifier). KzgAccumulator(P1, P2), which passes the pairing iff the proof's opening holds; for a valid proof it is
    (s W', W') with W' the proof's last point, the pair every correct SHPLONK verifier reaches. A ProofFailure("transcript", ...)
    when the bytes cannot be read. Spectre's inner snarks are written with poseidon.PoseidonTranscriptWrite, so pass
    transcript_read=poseidon.PoseidonTranscriptRead for them. One multiexp on be."""
    got = _opening_points(be, vp, vk, instances, proof, transcript_read)
    return got if isinstance(got, ProofFailure) else KzgAccumulator(*got)


def aggregate_accumulators(be, accs, transcript=None):
    """snark-verifier's KzgAs::create_proof as snark_verifier_sdk's aggregation calls it, without zk. One accumulator is
    returned as it is, whatever the transcript: that is Spectre's case, where each aggregation circuit wraps one snark. Several
    are folded into sum_i r^i accs[i], starting at r^0 = 1, with one multiexp per side; the result passes the pairing iff every
    input does, except with probability at most len(accs) / r. r is squeezed from `transcript` (default
    poseidon.PoseidonTranscriptWrite(0)) after it absorbs each lhs and rhs, in order, as common points.
    That framing is not pinned against snark-verifier, as poseidon.py's framing is not: snark-verifier squeezes r from the
    aggregation proof's own Poseidon transcript, which starts without the key digest this default absorbs. So for several
    accumulators r and the folded pair are this library's own."""
    accs = [KzgAccumulator(*a) for a in accs]
    if not accs:
        raise ValueError("aggregate_accumulators: no accumulator given")
    if len(accs) == 1:
        return accs[0]
    if transcript is None:
        transcript = poseidon.PoseidonTranscriptWrite(0)
    for a in accs:
        transcript.common_ec_point(a.lhs)
        transcript.common_ec_point(a.rhs)
    r = transcript.squeeze_challenge()
    powers = [pow(r, i, R_MOD) for i in range(len(accs))]
    return KzgAccumulator(_multiexp(be, powers, [a.lhs for a in accs]), _multiexp(be, powers, [a.rhs for a in accs]))


def evm_pairing_points(be, vp, vk, instances, proof, accumulator_indices):
    """The two G1 points the generated verifier contract hands to the pairing precompile (0x08) for an aggregation proof over
    the EVM transcript, with the r that combines them: (r, P1 + r lhs, P2 + r rhs). (P1, P2) are the SHPLONK opening's points,
    (lhs, rhs) the accumulator decoded from the instances at accumulator_indices, and r = keccak256(P1 || P2 || lhs || rhs)
    mod r_F over the 32-byte big-endian coordinates. The contract accepts iff e(P1 + r lhs, [1]_2) e(P2 + r rhs, -[s]_2) = 1,
    so this reproduces its decision before a transaction is sent. A ProofFailure ("transcript" or "accumulator_encoding")
    where the contract reverts before it gets that far. Three multiexps on be."""
    got = _replay(be, vp, vk, instances, proof, EvmTranscriptRead, accumulator_indices)
    if isinstance(got, ProofFailure):
        return got
    p1, p2, acc = got
    r = int.from_bytes(keccak256(b"".join(v.to_bytes(32, "big") for pt in (p1, p2, acc.lhs, acc.rhs) for v in pt)), "big") % R_MOD
    return r, _multiexp(be, [1, r], [p1, acc.lhs]), _multiexp(be, [1, r], [p2, acc.rhs])


_CHECK_FAILED = {"opening": "the SHPLONK opening fails its pairing check",
                 "accumulator": "the KZG accumulator in the instances fails its pairing check"}


def verify_proofs(be, vp, items, transcript_read=EvmTranscriptRead, accumulator_indices=None):
    """verify_proof for every (vk, instances, proof) of `items`; the keys may differ (step and committee-update proofs together).
    One verdict per item, in verify_proof's form: None for an accepted proof, else a ProofFailure. An item may carry a fourth
    element, its accumulator indices, which then stand in for `accumulator_indices`: step and aggregation proofs share a batch.
    Every proof that gets past its transcript and accumulator encoding costs one multiexp, and all of them are decided by ONE
    pairing_check_batch call of m = 2 pairs per check: one check per proof, and a second for each aggregation proof.
    be: anything with best_multiexp(coeffs, bases) and pairing_check_batch(ps, qs, m) in the layouts of halo2.Backend; vp: a
    halo2.ParamsVerifierKZG."""
    verdicts, todo, ps, qs = [], [], [], []
    neg_s_g2 = _neg_g2(vp.s_g2)
    for item in items:
        vk, instances, proof = item[:3]
        indices = item[3] if len(item) > 3 else accumulator_indices
        got = _replay(be, vp, vk, instances, proof, transcript_read, indices)
        if isinstance(got, ProofFailure):
            verdicts.append(got)
            continue
        verdicts.append(None)
        p1, p2, acc = got
        checks = [("opening", p1, p2)] + ([] if acc is None else [("accumulator", acc.lhs, acc.rhs)])
        for kind, a, b in checks:
            todo.append((len(verdicts) - 1, kind))
            ps += [_g1_limbs(a), _g1_limbs(b)]
            qs += [vp.g2, neg_s_g2]
    if todo:
        ok = be.pairing_check_batch(np.stack(ps), np.stack(qs), 2)
        for (i, kind), good in zip(todo, ok):
            if not good and verdicts[i] is None:               # the opening's check comes first: the first failure is reported
                verdicts[i] = ProofFailure(kind, _CHECK_FAILED[kind])
    return verdicts


def verify_proof(be, vp, vk, instances, proof, transcript_read=EvmTranscriptRead, accumulator_indices=None):
    """halo2_proofs::plonk::verify_proof with VerifierSHPLONK and SingleStrategy: None when the proof is accepted, else a
    ProofFailure. instances: per instance column a list of ints (a wrong column count raises ValueError, a caller error as
    upstream's Error::InvalidInstances). transcript_read: EvmTranscriptRead (default) or poseidon.PoseidonTranscriptRead, the
    reading side of the transcript create_proof wrote. The final check is one pairing_check_batch call of one check.
    accumulator_indices: for an aggregation proof (AGGREGATION_ACCUMULATOR_INDICES for Spectre's), also decide the KZG
    accumulator in its instances as the verifier contract does, in the same pairing call; indices outside the instances raise
    ValueError. None (default) checks the proof alone, as halo2's verify_proof does."""
    return verify_proofs(be, vp, [(vk, instances, proof)], transcript_read, accumulator_indices)[0]
