"""Shared pieces of the verifier tests (tests/test_verify_cpu.py, tests/test_gpu_verify.py): the verifier params taken only from
the verifier contracts' constants, the committed fixtures with the alterations the contract rejected, and a pure-Python
stand-in for the two device calls spectre_b200.plonk.verify_proof makes."""
import glob
import json
import os

import numpy as np

from spectre_b200 import circuits, halo2, plonk
from tests import pypairing as pp
from tests import pyref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class PyBackend:
    """best_multiexp (pyref.msm) and pairing_check_batch (pypairing) in halo2.Backend's layouts"""

    def best_multiexp(self, coeffs, bases):
        scalars = [plonk.fr_int(r) for r in np.asarray(coeffs, dtype=np.uint64).reshape(-1, 4)]
        pts = [pyref.aff_tuple(tuple(pp.fq_ints(b))) for b in np.asarray(bases, dtype=np.uint64).reshape(-1, 8)]
        acc = pyref.msm(scalars, [p for p in pts])
        return pp.fq_limbs([0, 1, 0] if acc is None else [acc[0], acc[1], 1]).reshape(12)

    def pairing_check_batch(self, ps, qs, m):
        ps = np.asarray(ps, dtype=np.uint64).reshape(-1, 8)
        qs = np.asarray(qs, dtype=np.uint64).reshape(-1, 16)
        g1 = [pyref.aff_tuple(tuple(pp.fq_ints(p))) for p in ps]
        g2 = [pp.g2_from_limbs(q) for q in qs]
        return [pp.pairing_check(g1[j:j + m], g2[j:j + m]) for j in range(0, len(g1), m)]


def _g2_from_contract(words):
    """a G2 point as the verifier contracts store it: x.c1, x.c0, y.c1, y.c0"""
    x1, x0, y1, y0 = [int(v, 16) for v in words]
    return ((x0, x1), (y0, y1))


def contract_g2(kats):
    """([1]_2, [s]_2) from the contract constants alone: g2_generator, and -[s]_2 with y negated"""
    g2 = _g2_from_contract(kats["g2_generator"]["x_c1,x_c0,y_c1,y_c0"])
    neg_s = _g2_from_contract(kats["neg_s_g2_sync_step"]["x_c1,x_c0,y_c1,y_c0"])
    return g2, pp.g2_neg(neg_s)


def contract_vp(kats, s_g2=None):
    g1 = tuple(int(v, 16) for v in kats["g1_generator"]["xy"])
    g2, s = contract_g2(kats)
    return halo2.ParamsVerifierKZG(pp.g1_limbs(g1), pp.g2_limbs(g2), pp.g2_limbs(s if s_g2 is None else s_g2))


def fixtures():
    return sorted(glob.glob(os.path.join(GOLDEN, "aggregation_k*_proof.json")))


def load_fixture(path):
    """(vk, instances, proof, the contract's own VK points) of a committed fixture"""
    with open(path) as f:
        fx = json.load(f)
    with open(os.path.join(GOLDEN, "verifier_contract_runs.json")) as f:
        run = json.load(f)[os.path.basename(path)]
    pts = [(int(x, 16), int(y, 16)) for x, y in fx["vk_points"]]
    own = [(int(x, 16), int(y, 16)) for x, y in run["contract_vk_points"]]
    vk = plonk.VerifyingKey(circuits.aggregation_shape(), fx["k"], int(fx["vk_digest"]), pts[:4], pts[4:])
    return vk, [[int(v, 16) for v in fx["instances"]]], bytes.fromhex(fx["proof"]), own


def alterations(kats, vk, instances, proof, own):
    """the four changes the reference's verifier contract rejected: (name, vp, vk, instances, proof)"""
    vp = contract_vp(kats)
    bad = bytearray(proof); bad[11 * 64 - 1 + 32 * 3] ^= 1             # one bit of an evaluation
    g2, s = contract_g2(kats)
    return [("flipped_evaluation_bit", vp, vk, instances, bytes(bad)),
            ("changed_public_input", vp, vk, [instances[0][:-1] + [instances[0][-1] + 1]], proof),
            ("contract_vk_points", vp, vk._replace(fixed_commitments=own[:4], sigma_commitments=own[4:]), instances, proof),
            ("wrong_tau", contract_vp(kats, pp.g2_add(s, g2)), vk, instances, proof)]
