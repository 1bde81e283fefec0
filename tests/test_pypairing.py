"""CPU-only: the pure-Python pairing reference (tests/pypairing.py) is a pairing. Bilinear at random scalars, non-degenerate,
of order r, and e(tau G1, G2) = e(G1, s_g2) on the seed-0 SRS whose s_g2 the oracle computes. Its G2 generator is the verifier
contracts' own."""
import random

from tests import pypairing as pp
from tests import pyref
from tests.verify_common import contract_g2


def test_bilinear_at_random_scalars():
    rng = random.Random(71)
    e = pp.pairing(pp.G1_GEN, pp.G2_GEN)
    a, b = rng.randrange(1, pp.R), rng.randrange(1, pp.R)
    assert pp.pairing(pyref.ec_mul(pp.G1_GEN, a), pp.g2_mul(pp.G2_GEN, b)) == pp.f12_pow(e, a * b % pp.R)


def test_non_degenerate_and_of_order_r():
    e = pp.pairing(pp.G1_GEN, pp.G2_GEN)
    assert e != pp.F12_ONE
    assert pp.f12_pow(e, pp.R) == pp.F12_ONE


def test_seed0_srs_g2_trailer_holds_tau(orc, kats):
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    s_g2 = pp.g2_from_limbs(orc.srs_s_g2())
    assert pp.g2_on_curve(s_g2)
    assert pp.pairing(pyref.ec_mul(pp.G1_GEN, tau), pp.G2_GEN) == pp.pairing(pp.G1_GEN, s_g2)
    assert contract_g2(kats)[0] == pp.G2_GEN
