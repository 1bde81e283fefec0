#!/usr/bin/env python3
"""One-off (build container, ~25 GiB, ~15 min): run the COMPILED driver (include/spectre_b200_prover.hpp over the test-only
ABI shim) on the K = 23 fixture's circuit, witness and RNG stream and compare its proof with
tests/golden/aggregation_k23_proof.json -- the bytes the reference's verifier contract accepted.
The RNG stream is regenerated from the fixture's seed by replaying the driver's draw sizes (no second Python proof needed)."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as orc  # noqa: E402
from spectre_b200 import circuits  # noqa: E402
from tests.plonk_oracle_engine import SeededRng  # noqa: E402
from tests.test_cpp_prover import _build_shim_and_main  # noqa: E402


def main():
    path = os.path.join(ROOT, "tests", "golden", sys.argv[1] if len(sys.argv) > 1 else "aggregation_k23_proof.json")
    with open(path) as f:
        fx = json.load(f)
    k, n = fx["k"], 1 << fx["k"]
    instances = [int(v, 16) for v in fx["instances"]]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, fx["lookup_bits"], fx["groups"], seed=fx["seed"])
    bf = cs.blinding_factors()
    # create_proof's draw sizes for this shape (1 advice column, 1 lookup, 1 permutation set, degree 5), in order
    counts = [bf + 1, 1, bf + 1, bf + 1, 2, bf, 1, bf, 1, n, 1, cs.degree() - 1]
    rng = SeededRng(fx["seed"])
    exe = _build_shim_and_main()
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "meta.txt"), "w") as f:
            f.write("shape aggregation\nk %d\ndigest %x\ninstances %s\n" % (k, int(fx["vk_digest"]), " ".join("%x" % v for v in instances)))
            for (c1, r1), (c2, r2) in copies:
                f.write("copy %d %d %d %d\n" % (c1, r1, c2, r2))
            f.write("rng " + " ".join(str(c) for c in counts) + "\n")
        np.concatenate(fixed).tofile(os.path.join(d, "fixed.bin")); adv.tofile(os.path.join(d, "advice.bin"))
        with open(os.path.join(d, "rng.bin"), "wb") as f:
            for c in counts:
                f.write(rng(c).tobytes())
        orc.srs_tau().tofile(os.path.join(d, "tau.bin"))
        del fixed, adv
        t0 = time.time()
        out = subprocess.run([exe, d], capture_output=True, text=True)
        print(out.stdout.strip(), out.stderr.strip(), "%.0f s" % (time.time() - t0), flush=True)
        assert out.returncode == 0
        with open(os.path.join(d, "proof.bin"), "rb") as f:
            proof = f.read()
    same = proof.hex() == fx["proof"]
    print("compiled driver reproduces %s: %s" % (os.path.basename(path), same))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
