"""The oracle engine (tests/plonk_oracle_engine.py) with the engine methods a per-part proof calls -- TEST INFRASTRUCTURE.
Each is restated from the oracle's whole-coset routines, independently of the library's part kernels:
  * coeff_to_extended_part_many: the oracle's whole extended coset sliced [part::R];
  * extended_part_scatter: numpy strided assignment;
  * permutation_constraints with a coset generator: the oracle's permutation terms, reparametrised (below)."""
import numpy as np

from oracle import oracle as orc
from spectre_b200.plonk import ZETA
from tests.plonk_oracle_engine import OracleEngine


def permutation_constraints_coset(values, rot_scale, last_rotation, chunk_len, z, col_values, sigma, l0, l_last, l_active, beta, gamma, y, coset_generator,
                                  omega):
    """The permutation terms with X = coset_generator * omega^idx at row idx. The oracle's routine reads X as zeta * w^idx and
    starts delta^j beta X at beta * zeta; called with w = omega, beta' = beta * g / zeta and sigma' = sigma * zeta / g, its
    beta' X is beta g omega^idx and its beta' sigma' is beta sigma, so every term is the same field element."""
    zeta = orc.fr([ZETA])[0]
    g_inv, zeta_inv = orc.batch_invert(np.stack([coset_generator, zeta]))
    beta2 = orc.fr_binop("fr_mul", orc.fr_binop("fr_mul", beta, coset_generator), zeta_inv)
    ratio = orc.fr_binop("fr_mul", zeta, g_inv)
    sigma2 = [orc.vec_scale(s, ratio) for s in sigma]
    return orc.permutation_constraints(values, rot_scale, last_rotation, chunk_len, z, col_values, sigma2, l0, l_last, l_active, beta2, gamma, y, omega)


class PerPartOracleEngine(OracleEngine):
    def coeff_to_extended_part_many(self, bufs, part, outs):
        """coset part `part`: the whole extended coset sliced [part::R]"""
        R = 1 << (self.extended_k - self.k)
        for b, o in zip(bufs, outs):
            o.a[:] = self.dom.coeff_to_extended(b.a)[part::R]

    def extended_part_scatter(self, part_buf, part, values):
        values.a[part::1 << (self.extended_k - self.k)] = part_buf.a

    def zero(self, b):
        b.a[:] = 0

    def permutation_constraints(self, values, size, rot_scale, last_rotation, chunk_len, z, cols, sigma, l0, l_last, l_active, beta, gamma, y, ext_omega,
                                coset_generator=None):
        if coset_generator is None:
            return super().permutation_constraints(values, size, rot_scale, last_rotation, chunk_len, z, cols, sigma, l0, l_last, l_active, beta, gamma, y,
                                                   ext_omega)
        values.a[:] = permutation_constraints_coset(values.a, rot_scale, last_rotation, chunk_len, [b.a for b in z], [b.a for b in cols], [b.a for b in sigma],
                                                    l0.a, l_last.a, l_active.a, beta, gamma, y, coset_generator, ext_omega)
