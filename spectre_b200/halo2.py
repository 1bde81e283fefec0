"""Host-side mirror of the halo2_proofs surface that Spectre's prover reaches on the create_proof hot path,
bound to libspectre_b200.so through its C ABI (include/spectre_b200.h) with ctypes.

The names, argument meaning and failure behaviour follow the upstream Rust items so parity tests read like
the reference's own use of them (reference call sites: lightclient-circuits/src/util/circuit.rs:11-16,131,158,
177,211,263; prover/src/prover.rs:9-13,55):

    halo2_proofs::arithmetic::best_fft            -> best_fft(a, omega, log_n)
    halo2_proofs::arithmetic::best_multiexp       -> best_multiexp(coeffs, bases)
    halo2_proofs::poly::EvaluationDomain          -> EvaluationDomain(j, k)
    halo2_proofs::poly::kzg::commitment::ParamsKZG-> ParamsKZG.setup / .from_parts / .read_custom / .commit / .commit_lagrange
    arithmetic::{eval_polynomial, kate_division}, ff::BatchInvert -> same names
    halo2curves::bn256 multi_miller_loop + final_exponentiation -> Backend.pairing / Backend.pairing_check_batch
    halo2_proofs::poly::kzg::commitment::ParamsVerifierKZG -> ParamsVerifierKZG, ParamsKZG.verifier_params

Field elements are numpy uint64 arrays (..., 4) holding halo2curves' in-memory Montgomery limbs; G1Affine is
(..., 8) = x‖y with identity (0,0); G1 (Jacobian) is (12,) = x‖y‖z.

This is the real Rust binding's stand-in (no cargo in this image; INTEGRATION.md has the Rust `extern "C"`
block). There is NO CPU fallback: importing works anywhere, but creating a Backend without the built
library or without a CUDA device raises.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SPB_LIB_PATH") or os.path.join(_HERE, "libspectre_b200.so")   # SPB_LIB_PATH: A/B builds (tools/), never the product default

# BN254: r is the order of G1 and the modulus of the scalar field Fr, p the modulus of the base field Fq, and G1 is
# y^2 = x^3 + 3 over Fq. An element of either field is held as the four little-endian 64-bit limbs of its Montgomery form
# a 2^256 mod the modulus.
R_MOD = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
P_MOD = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
MONT_RADIX = 1 << 256
FQ_MONT_INV = pow(MONT_RADIX, -1, P_MOD)


def g1_on_curve(x, y):
    """x and y are canonical Fq ints (below p) and (x, y) lies on y^2 = x^3 + 3; the identity (0, 0) does not"""
    return x < P_MOD and y < P_MOD and (y * y - x * x * x - 3) % P_MOD == 0


BASIS_G = 0
BASIS_G_LAGRANGE = 1

ERR_DATA = -6                                                     # SPB_ERR_DATA: invalid input data
SERDE_FORMATS = {"RawBytes": 1, "RawBytesUnchecked": 2}          # SPB_SERDE_RAW_BYTES, SPB_SERDE_RAW_BYTES_UNCHECKED


class BackendError(RuntimeError):
    pass


_lib = None


def load_library():
    """dlopen the C-ABI library. Raises if it has not been built (python -m spectre_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise BackendError("libspectre_b200.so is not built (run `python -m spectre_b200.build`); there is no CPU fallback")
        lib = ctypes.CDLL(LIB_PATH)
        lib.spb_init.restype = ctypes.c_void_p
        lib.spb_init.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.spb_last_error.restype = ctypes.c_char_p
        lib.spb_last_error.argtypes = [ctypes.c_void_p]
        lib.spb_kernel_launches.restype = ctypes.c_uint64
        lib.spb_kernel_launches.argtypes = [ctypes.c_void_p]
        lib.spb_last_device_ms.restype = ctypes.c_float
        lib.spb_last_device_ms.argtypes = [ctypes.c_void_p]
        if hasattr(lib, "spb_last_msm_adds"):
            lib.spb_last_msm_adds.restype = ctypes.c_uint64
            lib.spb_last_msm_adds.argtypes = [ctypes.c_void_p]
        lib.spb_domain_extended_k.restype = ctypes.c_uint32
        lib.spb_domain_extended_k.argtypes = [ctypes.c_void_p]
        _lib = lib
    return _lib


def _p(a):
    if a is None:
        return None
    if isinstance(a, int):
        return ctypes.c_void_p(a)
    return a.ctypes.data_as(ctypes.c_void_p)


def _fr_array(a, n=None):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if a.ndim == 1:
        a = a.reshape(-1, 4)
    assert a.shape[-1] == 4
    if n is not None:
        assert a.shape[0] == n, "length mismatch"
    return a


def _pair_arrays(ps, qs):
    ps = np.ascontiguousarray(ps, dtype=np.uint64).reshape(-1, 8)
    qs = np.ascontiguousarray(qs, dtype=np.uint64).reshape(-1, 16)
    if ps.shape[0] != qs.shape[0]:
        raise ValueError("pairing: %d G1 points but %d G2 points" % (ps.shape[0], qs.shape[0]))
    return ps, qs


class Backend:
    """One spb_ctx. `devices`: list of CUDA device ids driven by this process (default [0])."""

    def __init__(self, devices=None):
        self.lib = load_library()
        devices = list(devices) if devices is not None else [0]
        ids = (ctypes.c_int * len(devices))(*devices)
        self.ctx = self.lib.spb_init(ids, len(devices))
        if not self.ctx:
            raise BackendError("spb_init failed: no usable CUDA device (the library has no CPU fallback)")
        self.ctx = ctypes.c_void_p(self.ctx)
        self.devices = devices

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.spb_shutdown(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc, what):
        if rc != 0:
            raise BackendError("%s failed (%d): %s" % (what, rc, self.lib.spb_last_error(self.ctx).decode()))

    def release_workspace(self):
        """spb_release_workspace: free the cached workspaces and twiddle tables of every device"""
        self.check(self.lib.spb_release_workspace(self.ctx), "spb_release_workspace")

    def stream(self, dev_index=0):
        """cudaStream_t (int) every `_dev` call of that device is ordered on: enqueue the producers of device buffers there."""
        self.lib.spb_stream.restype = ctypes.c_void_p
        self.lib.spb_stream.argtypes = [ctypes.c_void_p, ctypes.c_int]
        s = self.lib.spb_stream(self.ctx, dev_index)
        if not s:
            raise BackendError("spb_stream: no stream for device index %d" % dev_index)
        return int(s)

    @property
    def kernel_launches(self):
        return int(self.lib.spb_kernel_launches(self.ctx))

    @property
    def last_device_ms(self):
        return float(self.lib.spb_last_device_ms(self.ctx))

    @property
    def last_msm_adds(self):
        return int(self.lib.spb_last_msm_adds(self.ctx))

    @property
    def last_msm_stage_ms(self):
        out = (ctypes.c_float * 7)()
        self.lib.spb_last_msm_stage_ms(self.ctx, out)
        return dict(zip(("digits", "sort", "offsets", "accumulate", "stitch", "groups", "rowcol_weighted"), [float(v) for v in out]))

    def msm_geometry(self, n, tables=False):
        c = ctypes.c_uint32(); w = ctypes.c_uint32()
        self.lib.spb_msm_geometry(ctypes.c_size_t(n), ctypes.c_int(1 if tables else 0), ctypes.byref(c), ctypes.byref(w))
        return c.value, w.value

    # ---- arithmetic::best_fft --------------------------------------------------------------------------
    def best_fft(self, a, omega, log_n):
        """In-place on a copy; returns the transformed array. Panics (AssertionError) like upstream when
        a.len() != 1 << log_n."""
        a = _fr_array(a).copy()
        assert a.shape[0] == 1 << log_n, "best_fft: a.len() != 1 << log_n"
        omega = _fr_array(omega, 1)
        self.check(self.lib.spb_ntt(self.ctx, _p(a), ctypes.c_uint32(log_n), _p(omega)), "spb_ntt")
        return a

    def best_fft_dev(self, d_ptr, omega, log_n):
        omega = _fr_array(omega, 1)
        self.check(self.lib.spb_ntt_dev(self.ctx, _p(d_ptr), ctypes.c_uint32(log_n), _p(omega)), "spb_ntt_dev")

    # ---- arithmetic::best_multiexp ---------------------------------------------------------------------
    def best_multiexp(self, coeffs, bases):
        coeffs = _fr_array(coeffs)
        bases = np.ascontiguousarray(bases, dtype=np.uint64).reshape(-1, 8)
        assert coeffs.shape[0] == bases.shape[0], "best_multiexp: coeffs.len() != bases.len()"
        out = np.empty(12, dtype=np.uint64)
        self.check(self.lib.spb_msm_raw(self.ctx, _p(coeffs), _p(bases), ctypes.c_size_t(coeffs.shape[0]), _p(out)), "spb_msm_raw")
        return out

    # ---- pairing (halo2curves bn256 engine) ------------------------------------------------------------
    def pairing(self, ps, qs):
        """prod_i e(ps[i], qs[i]) (spb_pairing): ps (n, 8) G1 affine as best_multiexp takes them, qs (n, 16) G2 affine as
        ParamsKZG.get_g2 returns them. Returns the 12 Fq values of Gt, (12, 4) Montgomery limbs in the order c0.c0.c0 ... c1.c2.c1.
        An invalid input raises BackendError naming it (SPB_ERR_DATA)."""
        ps, qs = _pair_arrays(ps, qs)
        out = np.empty((12, 4), dtype=np.uint64)
        self.check(self.lib.spb_pairing(self.ctx, _p(ps), _p(qs), ctypes.c_size_t(ps.shape[0]), _p(out)), "spb_pairing")
        return out

    def pairing_check_batch(self, ps, qs, m):
        """spb_pairing_check_batch: check j holds iff prod_{i<m} e(ps[j m + i], qs[j m + i]) == 1; a list of len(ps) / m bools"""
        ps, qs = _pair_arrays(ps, qs)
        if m <= 0 or ps.shape[0] % m:
            raise ValueError("pairing_check_batch: %d pairs do not split into checks of m = %d" % (ps.shape[0], m))
        n_checks = ps.shape[0] // m
        ok = np.zeros(max(n_checks, 1), dtype=np.int32)
        self.check(self.lib.spb_pairing_check_batch(self.ctx, _p(ps), _p(qs), ctypes.c_size_t(m), ctypes.c_size_t(n_checks), _p(ok)), "spb_pairing_check_batch")
        return [bool(v) for v in ok[:n_checks]]

    # ---- batch ops -------------------------------------------------------------------------------------
    def batch_invert(self, a):
        a = _fr_array(a).copy()
        self.check(self.lib.spb_batch_invert(self.ctx, _p(a), ctypes.c_size_t(a.shape[0])), "spb_batch_invert")
        return a

    def eval_polynomial(self, poly, point):
        poly = _fr_array(poly); point = _fr_array(point, 1)
        out = np.empty(4, dtype=np.uint64)
        self.check(self.lib.spb_eval_polynomial(self.ctx, _p(poly), ctypes.c_size_t(poly.shape[0]), _p(point), _p(out)), "spb_eval_polynomial")
        return out

    def kate_division(self, a, b):
        a = _fr_array(a); b = _fr_array(b, 1)
        q = np.empty((a.shape[0] - 1, 4), dtype=np.uint64)
        self.check(self.lib.spb_kate_division(self.ctx, _p(a), ctypes.c_size_t(a.shape[0]), _p(b), _p(q)), "spb_kate_division")
        return q

    def grand_product(self, a):
        a = _fr_array(a)
        z = np.empty_like(a)
        self.check(self.lib.spb_grand_product(self.ctx, _p(a), ctypes.c_size_t(a.shape[0]), _p(z)), "spb_grand_product")
        return z

    def vec_mul(self, a, b):
        a = _fr_array(a).copy(); b = _fr_array(b, a.shape[0])
        self.check(self.lib.spb_vec_mul(self.ctx, _p(a), _p(b), ctypes.c_size_t(a.shape[0])), "spb_vec_mul")
        return a

    def vec_axpy(self, y, alpha, x):
        y = _fr_array(y).copy(); x = _fr_array(x, y.shape[0]); alpha = _fr_array(alpha, 1)
        self.check(self.lib.spb_vec_axpy(self.ctx, _p(y), _p(alpha), _p(x), ctypes.c_size_t(y.shape[0])), "spb_vec_axpy")
        return y

    def vec_scale(self, a, alpha):
        a = _fr_array(a).copy(); alpha = _fr_array(alpha, 1)
        self.check(self.lib.spb_vec_scale(self.ctx, _p(a), _p(alpha), ctypes.c_size_t(a.shape[0])), "spb_vec_scale")
        return a

    # ---- device-resident batch ops (pointers are ints: addresses on device 0 of the context) ----------
    def lincomb_dev(self, d_ptrs, y, d_out, n):
        ptrs = (ctypes.c_void_p * len(d_ptrs))(*d_ptrs)
        self.check(self.lib.spb_lincomb_dev(self.ctx, ptrs, ctypes.c_size_t(len(d_ptrs)), _p(_fr_array(y, 1)), _p(d_out), ctypes.c_size_t(n)), "spb_lincomb_dev")

    def eval_polynomial_dev(self, d_poly, n, point):
        out = np.empty(4, dtype=np.uint64)
        self.check(self.lib.spb_eval_polynomial_dev(self.ctx, _p(d_poly), ctypes.c_size_t(n), _p(_fr_array(point, 1)), _p(out)), "spb_eval_polynomial_dev")
        return out

    def eval_polynomial_many_dev(self, d_polys, n, points):
        """[(device address, point (4,))...] -> (count, 4) evaluations, one launch"""
        count = len(d_polys)
        out = np.empty((count, 4), dtype=np.uint64)
        if count:
            ptrs = (ctypes.c_void_p * count)(*d_polys)
            pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(count, 4)
            self.check(self.lib.spb_eval_polynomial_many_dev(self.ctx, ptrs, ctypes.c_size_t(n), _p(pts), ctypes.c_size_t(count), _p(out)), "spb_eval_polynomial_many_dev")
        return out

    def fr_random_chacha_dev(self, seed, first, d_out, n):
        """d_out[i] = the (first + i)-th Fr::random draw of ChaCha20Rng::from_seed(seed) (seed: int or 32 bytes), made on the device"""
        if isinstance(seed, int):
            seed = seed.to_bytes(32, "little")
        assert len(seed) == 32
        self.check(self.lib.spb_fr_random_chacha_dev(self.ctx, ctypes.c_char_p(bytes(seed)), ctypes.c_uint64(first), _p(d_out), ctypes.c_size_t(n)), "spb_fr_random_chacha_dev")

    def kate_division_dev(self, d_a, n, b, d_q):
        self.check(self.lib.spb_kate_division_dev(self.ctx, _p(d_a), ctypes.c_size_t(n), _p(_fr_array(b, 1)), _p(d_q)), "spb_kate_division_dev")

    def batch_invert_dev(self, d_a, n):
        self.check(self.lib.spb_batch_invert_dev(self.ctx, _p(d_a), ctypes.c_size_t(n)), "spb_batch_invert_dev")

    def grand_product_dev(self, d_a, n, d_z):
        self.check(self.lib.spb_grand_product_dev(self.ctx, _p(d_a), ctypes.c_size_t(n), _p(d_z)), "spb_grand_product_dev")

    def product_dev(self, d_a, n):
        out = np.empty(4, dtype=np.uint64)
        self.check(self.lib.spb_product_dev(self.ctx, _p(d_a), ctypes.c_size_t(n), _p(out)), "spb_product_dev")
        return out

    def grand_product_seeded_dev(self, d_a, n, init, d_z):
        self.check(self.lib.spb_grand_product_seeded_dev(self.ctx, _p(d_a), ctypes.c_size_t(n), _p(_fr_array(init, 1)), _p(d_z)), "spb_grand_product_seeded_dev")

    def vec_mul_dev(self, d_a, d_b, n):
        self.check(self.lib.spb_vec_mul_dev(self.ctx, _p(d_a), _p(d_b), ctypes.c_size_t(n)), "spb_vec_mul_dev")

    def vec_scale_dev(self, d_a, alpha, n):
        self.check(self.lib.spb_vec_scale_dev(self.ctx, _p(d_a), _p(_fr_array(alpha, 1)), ctypes.c_size_t(n)), "spb_vec_scale_dev")

    # ---- quotient numerator (plonk::evaluation) ---------------------------------------------------------
    def graph_evaluate_dev(self, prog, ncalc, n_inter, constants, rotations, d_fixed, d_advice, d_instance, challenges, beta, gamma, theta, y,
                           d_values, size, rot_scale):
        """GraphEvaluator::evaluate for every extended row; column lists hold device addresses (ints)."""
        class _Graph(ctypes.Structure):
            _fields_ = [("program", ctypes.c_void_p), ("program_words", ctypes.c_size_t), ("num_calculations", ctypes.c_uint32),
                        ("num_intermediates", ctypes.c_uint32), ("constants", ctypes.c_void_p), ("num_constants", ctypes.c_uint32),
                        ("rotations", ctypes.c_void_p), ("num_rotations", ctypes.c_uint32)]
        prog = np.ascontiguousarray(prog, dtype=np.uint32); rotations = np.ascontiguousarray(rotations, dtype=np.int32)
        constants = np.ascontiguousarray(constants, dtype=np.uint64).reshape(-1, 4)
        challenges = np.ascontiguousarray(challenges, dtype=np.uint64).reshape(-1, 4)
        g = _Graph(prog.ctypes.data, prog.size, ncalc, n_inter, constants.ctypes.data, constants.shape[0], rotations.ctypes.data, rotations.size)
        mk = lambda ps: (ctypes.c_void_p * max(1, len(ps)))(*ps)
        self.check(self.lib.spb_graph_evaluate_dev(self.ctx, ctypes.byref(g), mk(d_fixed), len(d_fixed), mk(d_advice), len(d_advice), mk(d_instance), len(d_instance),
                                                   _p(challenges), challenges.shape[0], _p(_fr_array(beta, 1)), _p(_fr_array(gamma, 1)), _p(_fr_array(theta, 1)),
                                                   _p(_fr_array(y, 1)), _p(d_values), ctypes.c_uint64(size), ctypes.c_int32(rot_scale)), "spb_graph_evaluate_dev")

    def permutation_constraints_dev(self, d_values, size, rot_scale, last_rotation, chunk_len, d_z, d_col_values, d_sigma, d_l0, d_l_last, d_l_active,
                                    beta, gamma, y, extended_omega):
        mk = lambda ps: (ctypes.c_void_p * max(1, len(ps)))(*ps)
        self.check(self.lib.spb_permutation_constraints_dev(self.ctx, _p(d_values), ctypes.c_uint64(size), ctypes.c_int32(rot_scale), ctypes.c_int32(last_rotation),
                                                            len(d_z), chunk_len, mk(d_z), len(d_col_values), mk(d_col_values), mk(d_sigma), _p(d_l0), _p(d_l_last),
                                                            _p(d_l_active), _p(_fr_array(beta, 1)), _p(_fr_array(gamma, 1)), _p(_fr_array(y, 1)),
                                                            _p(_fr_array(extended_omega, 1))), "spb_permutation_constraints_dev")

    def permutation_constraints_coset_dev(self, d_values, size, rot_scale, last_rotation, chunk_len, d_z, d_col_values, d_sigma, d_l0, d_l_last, d_l_active,
                                          beta, gamma, y, coset_generator, omega):
        """permutation_constraints_dev with X = coset_generator * omega^idx at row idx (a coset part of the extended coset)"""
        mk = lambda ps: (ctypes.c_void_p * max(1, len(ps)))(*ps)
        self.check(self.lib.spb_permutation_constraints_coset_dev(self.ctx, _p(d_values), ctypes.c_uint64(size), ctypes.c_int32(rot_scale), ctypes.c_int32(last_rotation),
                                                                  len(d_z), chunk_len, mk(d_z), len(d_col_values), mk(d_col_values), mk(d_sigma), _p(d_l0), _p(d_l_last),
                                                                  _p(d_l_active), _p(_fr_array(beta, 1)), _p(_fr_array(gamma, 1)), _p(_fr_array(y, 1)),
                                                                  _p(_fr_array(coset_generator, 1)), _p(_fr_array(omega, 1))), "spb_permutation_constraints_coset_dev")

    def lookup_constraints_dev(self, d_values, size, rot_scale, d_product, d_permuted_input, d_permuted_table, d_table_value, d_l0, d_l_last, d_l_active,
                               beta, gamma, y):
        self.check(self.lib.spb_lookup_constraints_dev(self.ctx, _p(d_values), ctypes.c_uint64(size), ctypes.c_int32(rot_scale), _p(d_product), _p(d_permuted_input),
                                                       _p(d_permuted_table), _p(d_table_value), _p(d_l0), _p(d_l_last), _p(d_l_active), _p(_fr_array(beta, 1)),
                                                       _p(_fr_array(gamma, 1)), _p(_fr_array(y, 1))), "spb_lookup_constraints_dev")

    # ---- argument provers (plonk::{permutation,lookup}::prover, multiopen::shplonk) -----------------------
    def permutation_product_dev(self, k, d_values, d_sigma, first_col, beta, gamma, blinds, last_z, d_z):
        """permutation::Argument::commit for one set; returns the new last_z. blinds: (blinding_factors, 4) RNG draws."""
        mk = lambda ps: (ctypes.c_void_p * max(1, len(ps)))(*ps)
        blinds = np.ascontiguousarray(blinds, dtype=np.uint64).reshape(-1, 4)
        lz = _fr_array(last_z, 1).copy()
        self.check(self.lib.spb_permutation_product_dev(self.ctx, ctypes.c_uint32(k), mk(d_values), mk(d_sigma), ctypes.c_uint32(len(d_values)), ctypes.c_uint32(first_col),
                                                        _p(_fr_array(beta, 1)), _p(_fr_array(gamma, 1)), _p(blinds), ctypes.c_uint32(blinds.shape[0]), _p(lz), _p(d_z)),
                   "spb_permutation_product_dev")
        return lz.reshape(4)

    def lookup_product_dev(self, n, d_compressed_input, d_compressed_table, d_permuted_input, d_permuted_table, beta, gamma, blinds, d_z):
        blinds = np.ascontiguousarray(blinds, dtype=np.uint64).reshape(-1, 4)
        self.check(self.lib.spb_lookup_product_dev(self.ctx, ctypes.c_size_t(n), _p(d_compressed_input), _p(d_compressed_table), _p(d_permuted_input), _p(d_permuted_table),
                                                   _p(_fr_array(beta, 1)), _p(_fr_array(gamma, 1)), _p(blinds), ctypes.c_uint32(blinds.shape[0]), _p(d_z)), "spb_lookup_product_dev")

    def weighted_sum_dev(self, d_ptrs, weights, d_out, n):
        ptrs = (ctypes.c_void_p * len(d_ptrs))(*d_ptrs)
        w = np.ascontiguousarray(weights, dtype=np.uint64).reshape(len(d_ptrs), 4)
        self.check(self.lib.spb_weighted_sum_dev(self.ctx, ptrs, _p(w), ctypes.c_size_t(len(d_ptrs)), _p(d_out), ctypes.c_size_t(n)), "spb_weighted_sum_dev")

    def shplonk_begin_dev(self, params, n, sets, y, v):
        """ProverSHPLONK::create_proof up to the first commitment. sets: list of (points (m,4), [device addresses], evals (n_polys, m, 4)).
        Returns (h commitment, handle for shplonk_finish_dev)."""
        class _Set(ctypes.Structure):
            _fields_ = [("points", ctypes.c_void_p), ("n_points", ctypes.c_uint32), ("d_polys", ctypes.c_void_p), ("n_polys", ctypes.c_uint32), ("evals", ctypes.c_void_p)]
        keep = []
        arr = (_Set * len(sets))()
        for i, (points, d_polys, evals) in enumerate(sets):
            points = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 4)
            evals = np.ascontiguousarray(evals, dtype=np.uint64).reshape(len(d_polys), points.shape[0], 4)
            ptrs = (ctypes.c_void_p * len(d_polys))(*d_polys)
            keep += [points, evals, ptrs]
            arr[i] = _Set(points.ctypes.data, points.shape[0], ctypes.cast(ptrs, ctypes.c_void_p).value, len(d_polys), evals.ctypes.data)
        out = np.empty(12, dtype=np.uint64); h = ctypes.c_void_p()
        self.check(self.lib.spb_shplonk_begin_dev(self.ctx, params.h, ctypes.c_size_t(n), arr, ctypes.c_uint32(len(sets)), _p(_fr_array(y, 1)), _p(_fr_array(v, 1)),
                                                  _p(out), ctypes.byref(h)), "spb_shplonk_begin_dev")
        return out, h

    def shplonk_finish_dev(self, handle, u):
        """Consumes the handle, also when it raises."""
        out = np.empty(12, dtype=np.uint64)
        self.check(self.lib.spb_shplonk_finish_dev(self.ctx, handle, _p(_fr_array(u, 1)), _p(out)), "spb_shplonk_finish_dev")
        return out

    def shplonk_abort_dev(self, handle):
        """spb_shplonk_abort: release a handle of shplonk_begin_dev that will not be finished (its workspace goes back to the context)"""
        self.lib.spb_shplonk_abort.restype = None
        self.lib.spb_shplonk_abort(self.ctx, handle)

    def permute_expression_pair_dev(self, d_input, d_table, usable, d_permuted_input, d_permuted_table):
        """lookup::prover::permute_expression_pair on device buffers; raises like Error::ConstraintSystemFailure."""
        self.check(self.lib.spb_permute_expression_pair_dev(self.ctx, _p(d_input), _p(d_table), ctypes.c_size_t(usable), _p(d_permuted_input),
                                                            _p(d_permuted_table)), "spb_permute_expression_pair_dev")

    # ---- witness check (dev::MockProver::verify) ----------------------------------------------------------
    def nonzero_rows_dev(self, d_values, lo, hi, cap):
        """-> (the first `cap` rows r in [lo, hi) with values[r] != 0, ascending; their total number)"""
        rows, total = np.zeros(max(cap, 1), dtype=np.uint32), ctypes.c_uint64()
        self.check(self.lib.spb_nonzero_rows_dev(self.ctx, _p(d_values), ctypes.c_uint64(lo), ctypes.c_uint64(hi), ctypes.c_uint32(cap), _p(rows),
                                                 ctypes.byref(total)), "spb_nonzero_rows_dev")
        return [int(r) for r in rows[:min(cap, total.value)]], total.value

    def lookup_missing_rows_dev(self, d_input, d_table, usable, cap):
        """-> (the first `cap` rows r < usable whose input value is not among the table's usable rows, ascending; their total number)"""
        rows, total = np.zeros(max(cap, 1), dtype=np.uint32), ctypes.c_uint64()
        self.check(self.lib.spb_lookup_missing_rows_dev(self.ctx, _p(d_input), _p(d_table), ctypes.c_size_t(usable), ctypes.c_uint32(cap), _p(rows),
                                                        ctypes.byref(total)), "spb_lookup_missing_rows_dev")
        return [int(r) for r in rows[:min(cap, total.value)]], total.value

    def copy_mismatches_dev(self, k, d_values, d_sigma, usable, cap):
        """-> per permutation column: (its total of failing rows, [(row, col', row') of the first `cap`, ascending]).
        A sigma entry that labels no usable cell raises with ERR_DATA's text naming its column and row."""
        m = len(d_values)
        mk = lambda ps: (ctypes.c_void_p * max(1, len(ps)))(*ps)
        cells, totals = np.zeros((max(m * cap, 1), 4), dtype=np.uint32), np.zeros(max(m, 1), dtype=np.uint64)
        self.check(self.lib.spb_copy_mismatches_dev(self.ctx, ctypes.c_uint32(k), mk(d_values), mk(d_sigma), ctypes.c_uint32(m), ctypes.c_size_t(usable),
                                                    ctypes.c_uint32(cap), _p(cells), _p(totals)), "spb_copy_mismatches_dev")
        out = []
        for c in range(m):
            t = int(totals[c])
            out.append((t, [(int(r), int(c2), int(r2)) for _, r, c2, r2 in cells[c * cap:c * cap + min(cap, t)]]))
        return out

    # ---- proving-key check --------------------------------------------------------------------------------
    def fr_first_noncanonical_dev(self, d_elems, n):
        """-> the first index i < n whose stored limbs are not below r, or n when every element is canonical"""
        first = ctypes.c_uint64()
        self.check(self.lib.spb_fr_first_noncanonical_dev(self.ctx, _p(d_elems), ctypes.c_size_t(n), ctypes.byref(first)), "spb_fr_first_noncanonical_dev")
        return first.value

    def sigma_check_dev(self, k, d_sigma, usable, cap):
        """-> per permutation column: three (total, first `cap` rows ascending) for the kinds label, blinding, unlabelled"""
        m = len(d_sigma)
        ptrs = (ctypes.c_void_p * max(1, m))(*d_sigma)
        rows, totals = np.zeros(max(3 * m * cap, 1), dtype=np.uint32), np.zeros(max(3 * m, 1), dtype=np.uint64)
        self.check(self.lib.spb_sigma_check_dev(self.ctx, ctypes.c_uint32(k), ptrs, ctypes.c_uint32(m), ctypes.c_size_t(usable), ctypes.c_uint32(cap),
                                                _p(rows), _p(totals)), "spb_sigma_check_dev")
        out = []
        for c in range(m):
            kinds = []
            for q in range(3):
                t, j = int(totals[3 * c + q]), 3 * c + q
                kinds.append((t, [int(r) for r in rows[j * cap:j * cap + min(cap, t)]]))
            out.append(kinds)
        return out

    def vec_axpy_dev(self, d_y, alpha, d_x, n):
        """d_y[i] += alpha * d_x[i]"""
        self.check(self.lib.spb_vec_axpy_dev(self.ctx, _p(d_y), _p(_fr_array(alpha, 1)), _p(d_x), ctypes.c_size_t(n)), "spb_vec_axpy_dev")

    # ---- file <-> device streaming (params / proving-key files) -------------------------------------------
    def read_file_dev(self, path, offset, d_dst, nbytes):
        self.check(self.lib.spb_read_file_dev(self.ctx, path.encode(), ctypes.c_uint64(offset), _p(d_dst), ctypes.c_size_t(nbytes)), "spb_read_file_dev")

    def write_file_dev(self, path, d_src, nbytes, append=True):
        self.check(self.lib.spb_write_file_dev(self.ctx, path.encode(), ctypes.c_int(1 if append else 0), _p(d_src), ctypes.c_size_t(nbytes)), "spb_write_file_dev")

    # ---- utilities -------------------------------------------------------------------------------------
    def g1_fixed_base_mul(self, scalars):
        scalars = _fr_array(scalars)
        out = np.empty((scalars.shape[0], 8), dtype=np.uint64)
        self.check(self.lib.spb_g1_fixed_base_mul(self.ctx, _p(scalars), ctypes.c_size_t(scalars.shape[0]), _p(out)), "spb_g1_fixed_base_mul")
        return out

    TEST_FIELD_OPS = {"mul": 0, "add": 1, "sub": 2, "sqr": 3, "neg": 4, "dbl": 5, "inv": 6, "to_mont": 7, "from_mont": 8, "is_canonical": 9,
                      "pow": 10, "pow_u64": 11}
    TEST_CURVE_OPS = {"add_mixed": 0, "add": 1, "dbl": 2, "dbl_affine": 3, "to_affine": 4, "mul_u32": 5, "affine_check": 6}

    def test_field_op(self, field, op, a, b=None):
        """spb_test_field_op; b (exponent for pow / pow_u64) defaults to zeros for the unary ops"""
        a = _fr_array(a); b = np.zeros_like(a) if b is None else _fr_array(b, a.shape[0])
        out = np.empty_like(a)
        f = {"fr": 0, "fq": 1}[field]; o = self.TEST_FIELD_OPS[op]
        self.check(self.lib.spb_test_field_op(self.ctx, f, o, _p(a), _p(b), _p(out), ctypes.c_size_t(a.shape[0])), "spb_test_field_op")
        return out

    def test_field_mul_sub_mul(self, field, a, b, c, d):
        a = _fr_array(a); b, c, d = (_fr_array(x, a.shape[0]) for x in (b, c, d))
        out = np.empty_like(a)
        self.check(self.lib.spb_test_field_mul_sub_mul(self.ctx, {"fr": 0, "fq": 1}[field], _p(a), _p(b), _p(c), _p(d), _p(out), ctypes.c_size_t(a.shape[0])),
                   "spb_test_field_mul_sub_mul")
        return out

    def test_curve_op(self, op, p, q=None, k=None):
        """spb_test_curve_op on (n, 16) uint64 XYZZ points; q defaults to zeros, k (uint32 per point) is needed by mul_u32"""
        p = np.ascontiguousarray(p, dtype=np.uint64).reshape(-1, 16)
        q = np.zeros_like(p) if q is None else np.ascontiguousarray(q, dtype=np.uint64).reshape(-1, 16)
        assert q.shape == p.shape
        k = None if k is None else np.ascontiguousarray(k, dtype=np.uint32).reshape(p.shape[0])
        out = np.empty_like(p)
        self.check(self.lib.spb_test_curve_op(self.ctx, self.TEST_CURVE_OPS[op], _p(p), _p(q), _p(k), _p(out), ctypes.c_size_t(p.shape[0])), "spb_test_curve_op")
        return out

    def bench_modmul(self, field="fq", threads=132 * 2048, iters=2000, ilp=2):
        ms = ctypes.c_float(0)
        self.check(self.lib.spb_bench_modmul(self.ctx, {"fr": 0, "fq": 1}[field], ctypes.c_uint32(threads), ctypes.c_uint32(iters), ilp, ctypes.byref(ms)), "spb_bench_modmul")
        threads = (threads + 255) // 256 * 256
        return ms.value, threads * iters * (2 if ilp & 0x100 else ilp) / (ms.value * 1e-3)


class EvaluationDomain:
    """EvaluationDomain::<Fr>::new(j, k) ([UPSTREAM] halo2_proofs/src/poly/domain.rs)."""

    def __init__(self, backend, j, k):
        self.be = backend
        self.j, self.k = j, k
        h = ctypes.c_void_p()
        backend.check(backend.lib.spb_domain_new(backend.ctx, ctypes.c_uint32(j), ctypes.c_uint32(k), ctypes.byref(h)), "spb_domain_new")
        self.h = h
        self.extended_k = int(backend.lib.spb_domain_extended_k(h))
        c = np.empty((8, 4), dtype=np.uint64)
        backend.lib.spb_domain_constants(h, _p(c))
        (self.omega, self.omega_inv, self.extended_omega, self.extended_omega_inv, self.g_coset, self.g_coset_inv,
         self.ifft_divisor, self.extended_ifft_divisor) = [c[i].copy() for i in range(8)]

    def __del__(self):
        try:
            if self.be.ctx:
                self.be.lib.spb_domain_free(self.be.ctx, self.h)
        except Exception:
            pass

    def get_omega(self):
        return self.omega

    def extended_len(self):
        return 1 << self.extended_k

    def lagrange_to_coeff(self, a):
        a = _fr_array(a).copy()
        assert a.shape[0] == 1 << self.k
        self.be.check(self.be.lib.spb_lagrange_to_coeff(self.be.ctx, self.h, _p(a)), "spb_lagrange_to_coeff")
        return a

    def coeff_to_lagrange(self, a):
        a = _fr_array(a).copy()
        assert a.shape[0] == 1 << self.k
        self.be.check(self.be.lib.spb_coeff_to_lagrange(self.be.ctx, self.h, _p(a)), "spb_coeff_to_lagrange")
        return a

    def coeff_to_extended(self, a):
        a = _fr_array(a)
        assert a.shape[0] == 1 << self.k
        out = np.empty((1 << self.extended_k, 4), dtype=np.uint64)
        self.be.check(self.be.lib.spb_coeff_to_extended(self.be.ctx, self.h, _p(a), _p(out)), "spb_coeff_to_extended")
        return out

    def extended_to_coeff(self, a):
        a = _fr_array(a)
        assert a.shape[0] == 1 << self.extended_k
        out = np.empty(((1 << self.k) * (self.j - 1), 4), dtype=np.uint64)
        self.be.check(self.be.lib.spb_extended_to_coeff(self.be.ctx, self.h, _p(a), _p(out)), "spb_extended_to_coeff")
        return out

    # device-resident forms (int device addresses)
    def lagrange_to_coeff_dev(self, d_a):
        self.be.check(self.be.lib.spb_lagrange_to_coeff_dev(self.be.ctx, self.h, _p(d_a)), "spb_lagrange_to_coeff_dev")

    def lagrange_to_coeff_batch_dev(self, d_ptrs):
        ptrs = (ctypes.c_void_p * max(1, len(d_ptrs)))(*d_ptrs)
        self.be.check(self.be.lib.spb_lagrange_to_coeff_batch_dev(self.be.ctx, self.h, ptrs, ctypes.c_size_t(len(d_ptrs))), "spb_lagrange_to_coeff_batch_dev")

    def coeff_to_extended_batch_dev(self, d_in, d_out):
        pi = (ctypes.c_void_p * max(1, len(d_in)))(*d_in); po = (ctypes.c_void_p * max(1, len(d_out)))(*d_out)
        self.be.check(self.be.lib.spb_coeff_to_extended_batch_dev(self.be.ctx, self.h, pi, po, ctypes.c_size_t(len(d_in))), "spb_coeff_to_extended_batch_dev")

    def coeff_to_extended_part_batch_dev(self, part, d_in, d_out):
        """d_out[i] = rows part, part + R, part + 2R, ... of coeff_to_extended(d_in[i]) (2^k of them), R = 2^(extended_k - k)"""
        pi = (ctypes.c_void_p * max(1, len(d_in)))(*d_in); po = (ctypes.c_void_p * max(1, len(d_out)))(*d_out)
        self.be.check(self.be.lib.spb_coeff_to_extended_part_batch_dev(self.be.ctx, self.h, ctypes.c_uint32(part), pi, po, ctypes.c_size_t(len(d_in))),
                      "spb_coeff_to_extended_part_batch_dev")

    def extended_part_scatter_dev(self, part, d_part, d_extended):
        """d_extended[part + R m] = d_part[m] for m < 2^k"""
        self.be.check(self.be.lib.spb_extended_part_scatter_dev(self.be.ctx, self.h, ctypes.c_uint32(part), _p(d_part), _p(d_extended)),
                      "spb_extended_part_scatter_dev")

    def coeff_to_extended_dev(self, d_in, d_out):
        self.be.check(self.be.lib.spb_coeff_to_extended_dev(self.be.ctx, self.h, _p(d_in), _p(d_out)), "spb_coeff_to_extended_dev")

    def extended_to_coeff_dev(self, d_in, d_out):
        self.be.check(self.be.lib.spb_extended_to_coeff_dev(self.be.ctx, self.h, _p(d_in), _p(d_out)), "spb_extended_to_coeff_dev")

    def divide_by_vanishing_poly_dev(self, d_a):
        self.be.check(self.be.lib.spb_divide_by_vanishing_dev(self.be.ctx, self.h, _p(d_a)), "spb_divide_by_vanishing_dev")

    def divide_by_vanishing_poly(self, a):
        a = _fr_array(a).copy()
        assert a.shape[0] == 1 << self.extended_k
        self.be.check(self.be.lib.spb_divide_by_vanishing(self.be.ctx, self.h, _p(a)), "spb_divide_by_vanishing")
        return a


class ParamsKZG:
    """ParamsKZG<Bn256> with g and g_lagrange resident on the device(s)."""

    def __init__(self, backend, k, handle):
        self.be, self.k, self.n, self.h = backend, k, 1 << k, handle

    @classmethod
    def setup(cls, backend, k, s):
        """ParamsKZG::setup(k, rng) where `s` is the secret the rng would draw (Montgomery limbs)."""
        s = _fr_array(s, 1)
        h = ctypes.c_void_p()
        backend.check(backend.lib.spb_srs_setup(backend.ctx, ctypes.c_uint32(k), _p(s), ctypes.byref(h)), "spb_srs_setup")
        return cls(backend, k, h)

    @classmethod
    def from_parts(cls, backend, k, g=None, g_lagrange=None):
        """What ParamsKZG::read yields: upload the two bases (either may be None)."""
        n = 1 << k
        if g is not None:
            g = np.ascontiguousarray(g, dtype=np.uint64).reshape(-1, 8); assert g.shape[0] == n
        if g_lagrange is not None:
            g_lagrange = np.ascontiguousarray(g_lagrange, dtype=np.uint64).reshape(-1, 8); assert g_lagrange.shape[0] == n
        h = ctypes.c_void_p()
        backend.check(backend.lib.spb_srs_upload(backend.ctx, ctypes.c_uint32(k), _p(g), _p(g_lagrange), ctypes.byref(h)), "spb_srs_upload")
        return cls(backend, k, h)

    @classmethod
    def from_bases(cls, backend, bases):
        """Any n bases kept resident (spb_bases_upload): `multiexp(scalars)` is then best_multiexp(scalars, bases[:len(scalars)])
        without the 64 B x n upload spb_msm_raw pays per call. Only the monomial-basis slot of the handle is set."""
        bases = np.ascontiguousarray(bases, dtype=np.uint64).reshape(-1, 8)
        h = ctypes.c_void_p()
        backend.check(backend.lib.spb_bases_upload(backend.ctx, _p(bases), ctypes.c_size_t(bases.shape[0]), ctypes.byref(h)), "spb_bases_upload")
        obj = cls(backend, max(0, (bases.shape[0] - 1).bit_length()), h)
        obj.n = bases.shape[0]
        return obj

    def multiexp(self, scalars):
        """best_multiexp(scalars, the resident bases[:len(scalars)])"""
        return self._commit(BASIS_G, scalars)

    @classmethod
    def read(cls, backend, path):
        """Read a params file in the RawBytes layout (the params/kzg_bn254_{k}.srs cache of gen_srs) WITHOUT validating the
        points (spb_srs_read_file). Upstream's ParamsKZG::read checks them: that is read_custom(backend, path, "RawBytes")."""
        h = ctypes.c_void_p()
        backend.check(backend.lib.spb_srs_read_file(backend.ctx, path.encode(), ctypes.byref(h)), "spb_srs_read_file")
        return cls._from_read(backend, h)

    @classmethod
    def read_custom(cls, backend, path, format):
        """ParamsKZG::read_custom(reader, format). format "RawBytes": every coordinate must be canonical and every point on its
        curve, else BackendError naming the first invalid point (SPB_ERR_DATA, halo2's io::ErrorKind::InvalidData);
        "RawBytesUnchecked": no checks."""
        if format not in SERDE_FORMATS:
            raise ValueError("read_custom: format must be one of %s (the compressed Processed format is not implemented)" % sorted(SERDE_FORMATS))
        h = ctypes.c_void_p()
        backend.check(backend.lib.spb_srs_read_file_custom(backend.ctx, path.encode(), ctypes.c_int(SERDE_FORMATS[format]), ctypes.byref(h)),
                      "spb_srs_read_file_custom")
        return cls._from_read(backend, h)

    @classmethod
    def _from_read(cls, backend, h):
        backend.lib.spb_srs_k.restype = ctypes.c_uint32
        backend.lib.spb_srs_k.argtypes = [ctypes.c_void_p]
        return cls(backend, int(backend.lib.spb_srs_k(h)), h)

    def downsize(self, k):
        """ParamsKZG::downsize(k): a new handle with g truncated to 2^k points and g_lagrange = g_to_lagrange(g) recomputed on the
        device (upstream mutates in place; here the old handle stays valid until dropped)."""
        h = ctypes.c_void_p()
        self.be.check(self.be.lib.spb_srs_downsize(self.be.ctx, self.h, ctypes.c_uint32(k), ctypes.byref(h)), "spb_srs_downsize")
        return ParamsKZG(self.be, k, h)

    def contribute(self, t):
        """One powers-of-tau update by the secret t (Montgomery limbs, 0 < t < r; spb_srs_contribute): a new handle with g[j]
        t^j g[j], g_lagrange = g_to_lagrange of that g, and the trailer's s_g2 times t, all computed on the device(s). The handle
        needs its G2 trailer (set_g2) and no window tables; it stays valid and unchanged. plonk.contribute_params wraps this with
        the public record of the update."""
        t = _fr_array(t, 1)
        h = ctypes.c_void_p()
        self.be.check(self.be.lib.spb_srs_contribute(self.be.ctx, self.h, _p(t), ctypes.byref(h)), "spb_srs_contribute")
        return ParamsKZG(self.be, self.k, h)

    def write(self, path):
        self.be.check(self.be.lib.spb_srs_write_file(self.be.ctx, self.h, path.encode()), "spb_srs_write_file")

    def set_g2(self, g2, s_g2):
        g2 = np.ascontiguousarray(g2, dtype=np.uint64).reshape(16); s_g2 = np.ascontiguousarray(s_g2, dtype=np.uint64).reshape(16)
        self.be.check(self.be.lib.spb_srs_set_g2(self.be.ctx, self.h, _p(g2), _p(s_g2)), "spb_srs_set_g2")

    def get_g2(self):
        g2 = np.empty(16, dtype=np.uint64); s_g2 = np.empty(16, dtype=np.uint64)
        self.be.check(self.be.lib.spb_srs_get_g2(self.be.ctx, self.h, _p(g2), _p(s_g2)), "spb_srs_get_g2")
        return g2, s_g2

    def verifier_params(self):
        """ParamsKZG::verifier_params: what a KZG verifier needs, g[0] and the G2 trailer. A handle without G2 points (one made by
        setup, which does not compute them) raises ValueError: give them with set_g2 first."""
        g2, s_g2 = self.get_g2()
        if not g2.any() or not s_g2.any():
            raise ValueError("verifier_params: the params hold no G2 points; set_g2 first")
        return ParamsVerifierKZG(self.get_g(0, 1)[0], g2, s_g2)

    def __del__(self):
        try:
            if self.be.ctx:
                self.be.lib.spb_srs_free(self.be.ctx, self.h)
        except Exception:
            pass

    def _commit(self, basis, poly):
        poly = _fr_array(poly)
        assert poly.shape[0] <= self.n, "commit: polynomial longer than the SRS"
        out = np.empty(12, dtype=np.uint64)
        self.be.check(self.be.lib.spb_msm(self.be.ctx, self.h, basis, _p(poly), ctypes.c_size_t(poly.shape[0]), _p(out)), "spb_msm")
        return out

    def commit(self, poly, blind=None):
        """Params::commit (monomial basis); the blind is ignored, as in the KZG scheme upstream."""
        return self._commit(BASIS_G, poly)

    def commit_lagrange(self, poly, blind=None):
        return self._commit(BASIS_G_LAGRANGE, poly)

    def precompute(self):
        """Build the 2^(c*j) window tables of both bases (one-time, W x memory); later commits use one bucket set."""
        self.be.check(self.be.lib.spb_srs_precompute(self.be.ctx, self.h), "spb_srs_precompute")
        return self

    def commit_batch(self, basis, polys):
        """count commitments against one basis, pipelined over the library's stream lanes. polys: list of (n,4) host arrays."""
        polys = [_fr_array(p) for p in polys]
        n = polys[0].shape[0]
        assert all(p.shape[0] == n for p in polys) and n <= self.n
        ptrs = (ctypes.c_void_p * len(polys))(*[p.ctypes.data for p in polys])
        out = np.empty((len(polys), 12), dtype=np.uint64)
        self.be.check(self.be.lib.spb_msm_batch(self.be.ctx, self.h, basis, ptrs, ctypes.c_size_t(n), ctypes.c_size_t(len(polys)), _p(out)), "spb_msm_batch")
        return out

    def commit_batch_dev(self, basis, d_ptrs, n):
        ptrs = (ctypes.c_void_p * len(d_ptrs))(*d_ptrs)
        out = np.empty((len(d_ptrs), 12), dtype=np.uint64)
        self.be.check(self.be.lib.spb_msm_batch_dev(self.be.ctx, self.h, basis, ptrs, ctypes.c_size_t(n), ctypes.c_size_t(len(d_ptrs)), _p(out)), "spb_msm_batch_dev")
        return out

    def commit_dev(self, basis, d_ptr, n):
        out = np.empty(12, dtype=np.uint64)
        self.be.check(self.be.lib.spb_msm_dev(self.be.ctx, self.h, basis, _p(d_ptr), ctypes.c_size_t(n), _p(out)), "spb_msm_dev")
        return out

    def get_g(self, start=0, count=None, basis=BASIS_G):
        count = self.n - start if count is None else count
        out = np.empty((count, 8), dtype=np.uint64)
        self.be.check(self.be.lib.spb_srs_download(self.be.ctx, self.h, basis, ctypes.c_size_t(start), ctypes.c_size_t(count), _p(out)), "spb_srs_download")
        return out


class ParamsVerifierKZG:
    """ParamsVerifierKZG<Bn256> (upstream's name for the verifier's part of the params): g = g[0] (uint64[8], G1 affine),
    g2 = [1]_2 and s_g2 = [s]_2 (uint64[16] each, the params file's G2 trailer layout), all Montgomery limbs. Made by
    ParamsKZG.verifier_params, or directly from constants (a verifier contract's G2 words, say)."""

    def __init__(self, g, g2, s_g2):
        self.g = np.ascontiguousarray(g, dtype=np.uint64).reshape(8).copy()
        self.g2 = np.ascontiguousarray(g2, dtype=np.uint64).reshape(16).copy()
        self.s_g2 = np.ascontiguousarray(s_g2, dtype=np.uint64).reshape(16).copy()


def g1_sum(points):
    """Fold Jacobian points (n, 12) on the host: the multi-rank MSM epilogue after all_gather."""
    pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 12)
    out = np.empty(12, dtype=np.uint64)
    rc = load_library().spb_g1_sum(_p(pts), ctypes.c_size_t(pts.shape[0]), _p(out))
    if rc != 0:
        raise BackendError("spb_g1_sum failed (%d)" % rc)
    return out


def g1_sum_batch(points):
    """points: (groups, count, 12) Jacobian partial sums (row g = rank g's batch) -> (count, 12): one C call per batch."""
    pts = np.ascontiguousarray(points, dtype=np.uint64)
    groups, count = pts.shape[0], pts.shape[1]
    out = np.empty((count, 12), dtype=np.uint64)
    rc = load_library().spb_g1_sum_batch(_p(pts), ctypes.c_size_t(groups), ctypes.c_size_t(count), _p(out))
    if rc != 0:
        raise BackendError("spb_g1_sum_batch failed (%d)" % rc)
    return out


def jacobian_to_affine_ints(j):
    """(12,) Jacobian Montgomery limbs -> (x, y) canonical ints, identity -> (0, 0). Pure Python (for tests/logs)."""
    j = np.ascontiguousarray(j, dtype=np.uint64).reshape(3, 4)
    v = [(int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192) * FQ_MONT_INV % P_MOD for r in j]
    if v[2] == 0:
        return (0, 0)
    zi = pow(v[2], -1, P_MOD)
    return (v[0] * zi * zi % P_MOD, v[1] * zi * zi * zi % P_MOD)
