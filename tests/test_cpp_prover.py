"""CPU tests of the compiled host side (include/spectre_b200_prover.hpp): host field arithmetic, Keccak and the EVM
transcript against their Python counterparts."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from spectre_b200.transcript import EvmTranscriptWrite, keccak256
from tests import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hooks():
    so = os.path.join(ROOT, "tests", "cpp", "libprover_hooks.so")
    src = os.path.join(ROOT, "tests", "cpp", "prover_hooks.cpp")
    hdr = os.path.join(ROOT, "include", "spectre_b200_prover.hpp")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-o", so, src])
    return ctypes.CDLL(so)


def _u(v):
    return np.array([(v >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64)


def _i(a):
    return sum(int(a[i]) << (64 * i) for i in range(4))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("fq", [0, 1])
def test_host_field(hooks, fq):
    m = pyref.P_MOD if fq else pyref.R_MOD
    rng = random.Random(fq)
    vals = [0, 1, 2, m - 1, m - 2, (1 << 253) % m] + [rng.randrange(m) for _ in range(200)]
    out = np.zeros(4, dtype=np.uint64)
    for a, b in zip(vals, reversed(vals)):
        hooks.ph_mul(fq, _p(_u(a)), _p(_u(b)), _p(out)); assert _i(out) == a * b % m
        hooks.ph_add(fq, _p(_u(a)), _p(_u(b)), _p(out)); assert _i(out) == (a + b) % m
        hooks.ph_sub(fq, _p(_u(a)), _p(_u(b)), _p(out)); assert _i(out) == (a - b) % m
    for a in vals[1:40]:
        hooks.ph_inv(fq, _p(_u(a)), _p(out)); assert _i(out) * a % m == 1
        hooks.ph_pow(fq, _p(_u(a)), ctypes.c_uint64(12345678901), _p(out)); assert _i(out) == pow(a, 12345678901, m)


def test_keccak_and_transcript(hooks):
    rng = random.Random(9)
    for n in (0, 1, 31, 32, 135, 136, 137, 272, 1000):
        data = bytes(rng.randrange(256) for _ in range(n))
        out = (ctypes.c_uint8 * 32)()
        hooks.ph_keccak(data, ctypes.c_size_t(n), out)
        assert bytes(out) == keccak256(data)
    digest = rng.randrange(pyref.R_MOD)
    T = EvmTranscriptWrite(digest)
    ops, vals, chal = [], [], []
    g = (1, 2)
    for step in range(60):
        op = rng.choice([0, 1, 2, 3, 3])
        ops.append(op)
        if op == 0:
            v = rng.randrange(pyref.R_MOD); vals.append(v); T.common_scalar(v)
        elif op == 1:
            v = rng.randrange(pyref.R_MOD); vals.append(v); T.write_scalar(v)
        elif op == 2:
            pt = pyref.ec_mul(g, rng.randrange(1, pyref.R_MOD)); vals += [pt[0], pt[1]]; T.write_ec_point(pt)
        else:
            chal.append(T.squeeze_challenge())
    ops_a = np.array(ops, dtype=np.int32)
    vals_a = np.stack([_u(v) for v in vals])
    chal_a = np.zeros((len(chal), 4), dtype=np.uint64)
    proof = (ctypes.c_uint8 * 8192)(); absorbed = (ctypes.c_size_t * 64)()
    hooks.ph_transcript.restype = ctypes.c_size_t
    n = hooks.ph_transcript(_p(_u(digest)), _p(ops_a), ctypes.c_size_t(len(ops)), _p(vals_a), _p(chal_a), proof, absorbed)
    assert bytes(proof[:n]) == bytes(T.proof)
    assert [_i(c) for c in chal_a] == chal
    assert list(absorbed[:len(T.absorbed)]) == T.absorbed


def test_poseidon_permutation_and_transcript_twin(hooks):
    """The C++ PoseidonSpec / PoseidonTranscriptWrite against spectre_b200/poseidon.py: the permutation for t = 3 (incl. the
    reference implementation's known-answer vector) and t = 12, and a random transcript script (challenges and proof bytes)."""
    from spectre_b200 import poseidon
    state = np.stack([_u(v) for v in (0, 1, 2)])
    hooks.ph_poseidon_permute(3, 8, 57, _p(state))
    assert [_i(r) for r in state] == [0x115cc0f5e7d690413df64c6b9662e9cf2a3617f2743245519e19607a4417189a,
                                      0x0fca49b798923ab0239de1c9e7a4a9a2210312b6a2f616d18b5a87f9b628ae29,
                                      0x0e7ae82e40091e63cbd4f16a6d16310b3729d4b6e138fcf54110e2867045a30c]
    rng = random.Random(12)
    vals12 = [rng.randrange(pyref.R_MOD) for _ in range(12)]
    state = np.stack([_u(v) for v in vals12])
    hooks.ph_poseidon_permute(12, 8, 60, _p(state))
    assert [_i(r) for r in state] == poseidon.Spec(12, 8, 60).permute(vals12)
    digest = rng.randrange(pyref.R_MOD)
    T = poseidon.PoseidonTranscriptWrite(digest)
    ops, vals, chal = [], [], []
    for step in range(70):
        op = rng.choice([0, 1, 2, 3, 3])
        ops.append(op)
        if op == 0:
            v = rng.randrange(pyref.R_MOD); vals.append(v); T.common_scalar(v)
        elif op == 1:
            v = rng.randrange(pyref.R_MOD); vals.append(v); T.write_scalar(v)
        elif op == 2:
            pt = pyref.ec_mul((1, 2), rng.randrange(1, pyref.R_MOD)); vals += [pt[0], pt[1]]; T.write_ec_point(pt)
        else:
            chal.append(T.squeeze_challenge())
    ops_a = np.array(ops, dtype=np.int32)
    vals_a = np.stack([_u(v) for v in vals])
    chal_a = np.zeros((len(chal), 4), dtype=np.uint64)
    proof = (ctypes.c_uint8 * 8192)()
    hooks.ph_poseidon_transcript.restype = ctypes.c_size_t
    n = hooks.ph_poseidon_transcript(_p(_u(digest)), _p(ops_a), ctypes.c_size_t(len(ops)), _p(vals_a), _p(chal_a), proof)
    assert bytes(proof[:n]) == bytes(T.proof)
    assert [_i(c) for c in chal_a] == chal


# ---- the whole driver: C++ keygen + create_proof over the test-only ABI shim vs the Python driver on the oracle engine ------
def _build_shim_and_main():
    from oracle import oracle as orc
    orc.build()
    shim_dir = os.path.join(ROOT, "tests", "abi_shim")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    shim = os.path.join(shim_dir, "libspb_shim.so")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("spectre_b200.h", "spectre_b200_prover.hpp")]
    src = os.path.join(shim_dir, "shim.cpp")
    if not os.path.exists(shim) or os.path.getmtime(shim) < max(os.path.getmtime(p) for p in [src] + hdrs):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", shim, src, "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    exe = os.path.join(ROOT, "tests", "cpp", "prover_main")
    msrc = exe + ".cpp"
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(p) for p in [msrc, shim] + hdrs):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, msrc, "-L" + shim_dir, "-lspb_shim", "-Wl,-rpath," + shim_dir, "-L" + ref_dir, "-lhalo2_oracle",
                               "-Wl,-rpath," + ref_dir])
    return exe


class _RecordingRng:
    def __init__(self, inner, chacha_poly=None):
        self.inner, self.calls = inner, []
        if chacha_poly is not None:      # the bulk draw (random polynomial) comes from the engine's ChaCha20 stream, not from `inner`
            self.device_rows = lambda E, count: E.random_chacha(chacha_poly, 0, count)

    def __call__(self, count):
        out = self.inner(count)
        self.calls.append(np.ascontiguousarray(out, dtype=np.uint64).reshape(-1, 4))
        return out


@pytest.mark.parametrize("shape,k,chacha_poly,transcript", [("aggregation", 7, None, "evm"), ("halo2lib", 8, None, "evm"), ("aggregation", 7, bytes(range(32)), "evm"),
                                                          ("halo2lib", 8, None, "poseidon")])
def test_cpp_driver_reproduces_the_python_proof(orc, tmp_path, shape, k, chacha_poly, transcript):
    """include/spectre_b200_prover.hpp (keygen + create_proof in C++) over the test-only CPU shim of the C ABI produces the
    same VK commitments and the same proof bytes as spectre_b200/plonk.py on the oracle engine, from the same columns, copies
    and RNG stream -- also when the vanishing argument's random polynomial is drawn by the engine from a ChaCha20 seed
    (spb_fr_random_chacha_dev in the product) instead of arriving through the host rng."""
    from spectre_b200 import circuits, plonk
    from tests.plonk_oracle_engine import OracleEngine, SeededRng
    exe = _build_shim_and_main()
    instances = [7, 8, 9]
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, lookup_bits=3, groups=20)
        adv = [adv]; head = "shape aggregation"
    else:
        cs = circuits.halo2lib_shape(3, 2)
        fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=4, groups=20, num_gate_advice=3, num_lookup_advice=2)
        head = "shape halo2lib 3 2"
    digest = 0x1234567890abcdef1234
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest)
    rec = _RecordingRng(SeededRng(77), chacha_poly)
    if transcript == "poseidon":                                 # the inner snark's transcript: both drivers are transcript-agnostic
        from spectre_b200.poseidon import PoseidonTranscriptWrite as Tw
    else:
        Tw = EvmTranscriptWrite
    proof = plonk.create_proof(E, pk, [instances], adv, rec, Tw(pk.vk_digest))
    if chacha_poly is not None:
        assert (1 << k) not in [c.shape[0] for c in rec.calls]      # the n-row draw never went through the host stream
    d = str(tmp_path)
    with open(os.path.join(d, "meta.txt"), "w") as f:
        f.write(head + "\nk %d\ndigest %x\ninstances %s\n" % (k, digest, " ".join("%x" % v for v in instances)))
        for (c1, r1), (c2, r2) in copies:
            f.write("copy %d %d %d %d\n" % (c1, r1, c2, r2))
        f.write("rng " + " ".join(str(c.shape[0]) for c in rec.calls) + "\n")
        if chacha_poly is not None:
            f.write("chacha_poly %s\n" % chacha_poly.hex())
        f.write("transcript %s\n" % transcript)
    np.concatenate(fixed).tofile(os.path.join(d, "fixed.bin"))
    np.concatenate(adv).tofile(os.path.join(d, "advice.bin"))
    np.concatenate([c for c in rec.calls if c.shape[0]] or [np.zeros((0, 4), np.uint64)]).tofile(os.path.join(d, "rng.bin"))
    orc.srs_tau().tofile(os.path.join(d, "tau.bin"))
    out = subprocess.run([exe, d], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    with open(os.path.join(d, "vk.txt")) as f:
        vk = [(int(l[:64], 16), int(l[64:128], 16)) for l in f.read().split()]
    assert vk == pk.fixed_commitments + pk.sigma_commitments
    with open(os.path.join(d, "proof.bin"), "rb") as f:
        assert f.read() == proof


def _build_main_against_the_real_library(out_dir):
    from tools import cpp_driver
    return cpp_driver.build_main_against_the_real_library(str(out_dir))


def test_cpp_driver_links_against_the_real_library(tmp_path):
    """the same main builds with CudaMemory against libspectre_b200.so + cudart (every ABI symbol the driver uses exists there)"""
    assert os.path.exists(_build_main_against_the_real_library(tmp_path))


def _dump_case(*args):
    from tools import cpp_driver
    cpp_driver.dump_case(*args)


@pytest.mark.gpu
def test_cpp_driver_on_the_gpu_reproduces_the_oracle_proof(orc, tmp_path):
    """The compiled driver (include/spectre_b200_prover.hpp, CudaMemory on the context's stream) against libspectre_b200.so:
    the same proof bytes as the Python driver on the CPU oracle, proved twice in the same process."""
    from spectre_b200 import circuits, plonk
    from tests.plonk_oracle_engine import OracleEngine, SeededRng
    exe = _build_main_against_the_real_library(tmp_path)
    k, instances = 8, [7, 8, 9]
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, instances, lookup_bits=4, groups=20, num_gate_advice=3, num_lookup_advice=2)
    digest = 0x1234567890abcdef1234
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest)
    rec = _RecordingRng(SeededRng(77))
    proof = plonk.create_proof(E, pk, [instances], adv, rec, EvmTranscriptWrite(pk.vk_digest))
    d = str(tmp_path)
    _dump_case(d, "shape halo2lib 3 2", k, digest, instances, copies, [c.shape[0] for c in rec.calls], fixed, adv, [c for c in rec.calls if c.shape[0]], orc.srs_tau())
    out = subprocess.run([exe, d], capture_output=True, text=True, env=dict(os.environ, SPB_MAIN_REPEAT="2"))
    assert out.returncode == 0, out.stdout + out.stderr
    with open(os.path.join(d, "proof.bin"), "rb") as f:
        assert f.read() == proof


@pytest.mark.gpu
def test_cpp_driver_on_the_gpu_reproduces_the_contract_accepted_k23_fixture(orc, tmp_path):
    """K = 23: the compiled driver regenerates tests/golden/aggregation_k23_proof.json -- the bytes the reference's
    sync_step verifier contract accepted -- through the real library, with window tables, and prints its wall time
    (bench.py times the same binary)."""
    import json
    from spectre_b200 import circuits
    from tests.plonk_oracle_engine import SeededRng
    exe = _build_main_against_the_real_library(tmp_path)
    with open(os.path.join(ROOT, "tests", "golden", "aggregation_k23_proof.json")) as f:
        fx = json.load(f)
    k, n = fx["k"], 1 << fx["k"]
    instances = [int(v, 16) for v in fx["instances"]]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, instances, fx["lookup_bits"], fx["groups"], seed=fx["seed"])
    bf = cs.blinding_factors()
    counts = [bf + 1, 1, bf + 1, bf + 1, 2, bf, 1, bf, 1, n, 1, cs.degree() - 1]     # create_proof's draw sizes for this shape, in order
    rng = SeededRng(fx["seed"])
    d = str(tmp_path)
    _dump_case(d, "shape aggregation", k, int(fx["vk_digest"]), instances, copies, counts, fixed, [adv], [rng(c) for c in counts], orc.srs_tau())
    del fixed, adv
    out = subprocess.run([exe, d], capture_output=True, text=True, env=dict(os.environ, SPB_MAIN_REPEAT="2", SPB_MAIN_TABLES="1"))
    assert out.returncode == 0, out.stdout + out.stderr
    with open(os.path.join(d, "proof.bin"), "rb") as f:
        assert f.read().hex() == fx["proof"]
    ms = [float(l.split()[1]) for l in out.stdout.splitlines() if l.startswith("create_proof_ms")]
    print("compiled driver K=23 create_proof ms:", ms)
