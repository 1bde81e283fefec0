"""CPU binding of the proof driver's engine interface (spectre_b200/plonk.py) to the oracle -- TEST INFRASTRUCTURE.
The driver (protocol order, transcript, RNG) is shared; every numeric operation below is the oracle's restatement of
the upstream routine, so a proof produced through this engine is the CPU reference for the GPU engine's proof.
Commitments use the known-tau shortcut of the seed-0 SRS (commit(p) = p(tau) * G1), which is independent of any MSM."""
import numpy as np

from oracle import oracle as orc
from spectre_b200 import halo2


class Buf:
    def __init__(self, a):
        self.a = a


def _aff(pt8):
    x, y = orc.affine_ints(np.asarray(pt8).reshape(1, 8))[0]
    return (x, y)


class OracleEngine:
    def __init__(self, k, j):
        self.k, self.n = k, 1 << k
        self.dom = orc.Domain(j, k)
        self.extended_k = self.dom.extended_k

    def alloc(self, rows): return Buf(np.zeros((rows, 4), dtype=np.uint64))
    def upload(self, a): return Buf(np.ascontiguousarray(a, dtype=np.uint64).copy())
    def download(self, b): return b.a.copy()
    def clone(self, b): return Buf(b.a.copy())
    def view(self, b, lo, hi): return Buf(b.a[lo:hi])
    def write_rows(self, b, start, rows):
        rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, 4)
        b.a[start:start + rows.shape[0]] = rows
    def read_rows(self, b, start, count): return b.a[start:start + count].copy()
    def sync(self): pass
    def random_chacha(self, seed, first, rows): return Buf(orc.fr_random_chacha(rows, seed, first))
    def append_to_file(self, path, b, rows):
        with open(path, "ab") as f:
            f.write(np.ascontiguousarray(b.a[:rows], dtype=np.uint64).tobytes())
    def read_from_file(self, path, offset, rows):
        return Buf(np.fromfile(path, dtype=np.uint64, count=rows * 4, offset=offset).reshape(rows, 4).copy())

    def commit(self, basis, bufs, n):
        if basis == halo2.BASIS_G:
            return [_aff(orc.commit_known_tau(b.a[:n])) for b in bufs]
        return [_aff(orc.commit_lagrange_known_tau(self.k, b.a[:n])) for b in bufs]

    def lagrange_to_coeff(self, b): b.a[:] = self.dom.lagrange_to_coeff(b.a)
    def coeff_to_lagrange(self, b): b.a[:] = orc.best_fft(b.a, self.dom.omega, self.k)
    def coeff_to_extended(self, b): return Buf(self.dom.coeff_to_extended(b.a))
    def extended_to_coeff(self, e, rows):
        out = self.dom.extended_to_coeff(e.a)
        assert out.shape[0] == rows
        return Buf(out)
    def divide_by_vanishing(self, e): e.a[:] = self.dom.divide_by_vanishing_poly(e.a)

    def graph_evaluate(self, p, fixed, advice, instance, beta, gamma, theta, y, values, size, rot_scale):
        bgty = np.stack([beta, gamma, theta, y])
        values.a[:] = orc.graph_evaluate(p["prog"], p["ncalc"], p["ncalc"], p["constants"], p["rotations"], [b.a for b in fixed], [b.a for b in advice],
                                         [b.a for b in instance], np.zeros((1, 4), np.uint64), bgty, values.a, rot_scale)
    def permutation_constraints(self, values, size, rot_scale, last_rotation, chunk_len, z, cols, sigma, l0, l_last, l_active, beta, gamma, y, ext_omega):
        values.a[:] = orc.permutation_constraints(values.a, rot_scale, last_rotation, chunk_len, [b.a for b in z], [b.a for b in cols], [b.a for b in sigma],
                                                  l0.a, l_last.a, l_active.a, beta, gamma, y, ext_omega)
    def lookup_constraints(self, values, size, rot_scale, product, pin, ptab, table_value, l0, l_last, l_active, beta, gamma, y):
        values.a[:] = orc.lookup_constraints(values.a, rot_scale, product.a, pin.a, ptab.a, table_value.a, l0.a, l_last.a, l_active.a, beta, gamma, y)

    def permute_expression_pair(self, a, s, usable, out_a, out_s):
        pa, ps = orc.permute_expression_pair(a.a[:usable], s.a[:usable])
        out_a.a[:usable] = pa; out_s.a[:usable] = ps
    def permutation_product(self, values, sigma, first_col, beta, gamma, blinds, last_z, z):
        zz, lz = orc.permutation_product(self.k, [b.a for b in values], [b.a for b in sigma], first_col, beta, gamma, blinds, last_z)
        z.a[:] = zz
        return lz.reshape(4)
    def lookup_product(self, ci, ct, pi, pt, beta, gamma, blinds, z):
        z.a[:] = orc.lookup_product(ci.a, ct.a, pi.a, pt.a, beta, gamma, blinds)

    def eval_polynomial(self, b, n, point): return orc.eval_polynomial(b.a[:n], point)
    def lincomb(self, bufs, y, out, n): out.a[:n] = orc.vec_fold([b.a[:n] for b in bufs], y)
    def vec_scale(self, b, alpha, n): b.a[:n] = orc.vec_scale(b.a[:n], alpha)

    def shplonk_begin(self, sets, y, v):
        hs = [(pts, [b.a for b in polys], ev) for pts, polys, ev in sets]
        h_x = orc.shplonk_quotient(self.n, hs, y, v)
        return _aff(orc.commit_known_tau(h_x)), (hs, y, v, h_x)
    def shplonk_finish(self, state, u):
        hs, y, v, h_x = state
        return _aff(orc.commit_known_tau(orc.shplonk_linearisation(self.n, hs, y, v, u, h_x)))
    def shplonk_abort(self, state): pass                       # the state is host memory: nothing to release


class SeededRng:
    """Deterministic stand-in for the `rng: R` argument of create_proof: ChaCha20 Fr draws (the oracle's generator),
    consumed strictly in order so both engines see the same values at the same protocol positions."""

    def __init__(self, seed):
        self.seed, self.counter = seed, 0

    def __call__(self, count):
        if count == 0:
            return np.zeros((0, 4), dtype=np.uint64)
        self.counter += 1
        return orc.fr_random_chacha(count, (self.seed << 32) + self.counter)


class FailingTranscript:
    """An EvmTranscriptWrite that raises `exc` on its `fail_at`-th write_ec_point call (counting from 0); `fail_at=None` never
    raises and only counts. create_proof writes the SHPLONK h commitment as its second-to-last point and the opening as its last."""

    def __init__(self, vk_digest, fail_at=None, exc=RuntimeError):
        from spectre_b200.transcript import EvmTranscriptWrite
        self.inner, self.fail_at, self.exc, self.points = EvmTranscriptWrite(vk_digest), fail_at, exc, 0

    def write_ec_point(self, xy):
        if self.points == self.fail_at:
            raise self.exc("transcript failure injected at point %d" % self.points)
        self.points += 1
        return self.inner.write_ec_point(xy)

    def __getattr__(self, name):
        return getattr(self.inner, name)
