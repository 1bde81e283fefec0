"""A deterministic operand corpus for the device field primitives (spectre_b200/csrc/field.cuh), chosen by carry coverage.

Candidates come in families: special values (zero, one, m - 1 - i, 2^k mod m, all-ones and single limbs), structured limb
patterns (each limb one of 0, 1, 2^31, 2^32 - 1 or a modulus limb and its neighbours), exact and off-by-one product
differences for a*b - c*d, and uniform random operands. Every operand is a raw 256-bit integer below the modulus: the
primitives see limbs, not Montgomery meanings, so every expected value below is computed on the raw integers (a product is
a*b*2^-256 mod m).

The carry-trace build of the emulated PTX path (libhostemu_trace.so, ptx.cuh under SPB_EMULATE_PTX_TRACE) reports, per
source line and per instance on that line (the limbs of an unrolled loop), whether each CF-reading instruction saw CF = 0
and CF = 1 and what each discarded carry out was. A candidate is kept when it shows the trace an instance and value the kept
ones have not (greedy, in family order), so the corpus stays small and still drives every carry, limb by limb, that the
whole candidate set reaches. Everything is regenerated from fixed seeds in a few seconds.
"""
import ctypes
import functools
import os
import random
import subprocess

import numpy as np

from tests import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTEMU = os.path.join(ROOT, "tests", "hostemu")
FIELD_H = os.path.join(ROOT, "spectre_b200", "csrc", "field.cuh")

MODULI = {"fr": pyref.R_MOD, "fq": pyref.P_MOD}
FIELD_CODE = {"fr": 0, "fq": 1}
RINV = {f: pow(1 << 256, -1, m) for f, m in MODULI.items()}
# op codes of spb_test_field_op / he_field_op
OPS = {"mul": 0, "add": 1, "sub": 2, "sqr": 3, "neg": 4, "dbl": 5, "inv": 6, "to_mont": 7, "from_mont": 8, "is_canonical": 9, "pow": 10,
       "pow_u64": 11}
PRIMITIVES = ("mul", "sqr", "mul_sub_mul", "add", "sub", "neg", "from_mont")
ARITY = {"mul": 2, "sqr": 1, "mul_sub_mul": 4, "add": 2, "sub": 2, "neg": 1, "from_mont": 1}
M32 = 0xFFFFFFFF
TRACE_CF_IN0, TRACE_CF_IN1, TRACE_DROP0, TRACE_DROP1 = 1, 2, 4, 8


def expected(field, prim, ops):
    """the primitive's value on raw integer operands, as Python integers"""
    m, rinv = MODULI[field], RINV[field]
    a = ops[0]
    if prim == "mul":
        return a * ops[1] * rinv % m
    if prim == "sqr":
        return a * a * rinv % m
    if prim == "mul_sub_mul":
        return (a * ops[1] - ops[2] * ops[3]) * rinv % m
    if prim == "add":
        return (a + ops[1]) % m
    if prim == "sub":
        return (a - ops[1]) % m
    if prim == "neg":
        return -a % m
    if prim == "dbl":
        return 2 * a % m
    if prim == "from_mont":
        return a * rinv % m
    if prim == "to_mont":
        return (a << 256) % m
    if prim == "inv":                       # Montgomery inverse: (a R^-1)^-1 R = a^-1 R^2; inv(0) = 0
        return pow(a, -1, m) * pow(1 << 256, 2, m) % m if a else 0
    raise KeyError(prim)


# ---- candidate families ---------------------------------------------------------------------------------------------------
def _limbs32(v):
    return [(v >> (32 * j)) & M32 for j in range(8)]


def _below(v, m):
    return v if v < m else (v - m if v - m < m else v % m)


def special_values(m):
    """zero, one, m - 1 - i, 2^k mod m, all-ones / single / half-word limbs, and the values of the older carry-pattern tests"""
    F = (1 << 128) - 1
    v = [0, 1, 2, 3, m >> 1, (m >> 1) + 1, (m - 1) // 2, ((1 << 254) - 1) % m, (1 << 253) + 12345, F, F << 96, (F << 126) % m,
         ((1 << 126) - 1) << 128 | F, (m >> 128) << 128, m & F, F | (F >> 3) << 128, 0xFFFFFFFF00000000FFFFFFFF00000000FFFFFFFF00000000FFFFFFFF % m]
    v += [m - 1 - i for i in range(16)]
    v += [(1 << k) % m for k in range(256)]
    v += [(M32 << (32 * i)) % m for i in range(8)] + [((1 << (32 * i)) - 1) % m for i in range(1, 9)]
    v += [(1 << (32 * i)) % m for i in range(8)] + [(1 << (32 * i + 31)) % m for i in range(8)]
    out, seen = [], set()
    for x in v:
        x %= m
        if x not in seen:
            seen.add(x); out.append(x)
    return out


def structured_values(m, n, seed):
    """each 32-bit limb drawn from {0, 1, 2^31, 2^32 - 1, m_j - 1, m_j, m_j + 1} (m_j = the same limb of the modulus)"""
    rng = random.Random(seed)
    ml = _limbs32(m)
    out = []
    for _ in range(n):
        v = 0
        for j in range(8):
            v |= rng.choice([0, 1, 1 << 31, M32, (ml[j] - 1) & M32, ml[j], (ml[j] + 1) & M32]) << (32 * j)
        out.append(_below(v, m))
    return out


def random_values(m, n, seed):
    rng = random.Random(seed)
    return [rng.randrange(m) for _ in range(n)]


def _tuples(prim, pool, rng, n):
    k = ARITY[prim]
    if k == 1:
        return [(x,) for x in pool]
    return [tuple(rng.choice(pool) for _ in range(k)) for _ in range(n)]


def product_edges(m, seed):
    """a*b - c*d at its edges (integer level, raw operands): equal products, differences of +-1, and differences near
    -(m - 1)^2 (the most negative one: the borrow correction adds m * 2^256 to a value just above -m * 2^256)"""
    rng = random.Random(seed)
    out = []
    for _ in range(64):
        x, y, z = (rng.randrange(1, 1 << rng.choice((32, 64, 96, 126))) for _ in range(3))
        a, b = rng.randrange(m), rng.randrange(m)
        out += [(a, b, a, b), (a, b, b, a), (x * y % m, z, x, y * z % m) if x * y < m and y * z < m else (a, b, b, a)]
        c, d = rng.randrange(1, 1 << 127), rng.randrange(1, 1 << 127)
        for e in (1, -1):
            p = c * d + e
            out += [(1, p, c, d), (p, 1, d, c), (c, d, 1, p), (d, c, p, 1)]
        lo = rng.randrange(4)
        out += [(lo, rng.randrange(m), m - 1 - rng.randrange(4), m - 1 - rng.randrange(4)),
                (0, 0, m - 1 - rng.randrange(1 << 32), m - 1 - rng.randrange(1 << 32)),
                (rng.randrange(1 << 32), 1, rng.randrange(m), rng.randrange(m))]
    return out


def families(field, prim):
    """(name, candidate operand tuples) in the order the greedy selection visits them"""
    m = MODULI[field]
    rng = random.Random("%s/%s" % (field, prim))   # a str seed is hashed with SHA-512: independent of PYTHONHASHSEED
    spec = special_values(m)
    fams = []
    if ARITY[prim] == 1:
        fams.append(("special", [(x,) for x in spec]))
    elif ARITY[prim] == 2:
        fams.append(("special", [(x, y) for x in spec[:48] for y in spec[:48]] + _tuples(prim, spec, rng, 4000)))
    else:
        fams.append(("special", _tuples(prim, spec, rng, 4000)))
        fams.append(("product_edges", product_edges(m, 7)))
    fams.append(("structured", _tuples(prim, structured_values(m, 4000, 11), rng, 4000)))
    fams.append(("random", _tuples(prim, random_values(m, 4000, 13), rng, 4000)))
    return fams


# ---- the host-emulated libraries -----------------------------------------------------------------------------------------
VARIANTS = {"ptx": ["-DSPB_EMULATE_PTX"], "native": [], "trace": ["-DSPB_EMULATE_PTX", "-DSPB_EMULATE_PTX_TRACE"]}


def build_hostemu(out_dir, variant):
    """libhostemu_<variant>.so from tests/hostemu/hostemu.cpp, built into out_dir (the checkout may be read-only)"""
    so = os.path.join(str(out_dir), "libhostemu_%s.so" % variant)
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + VARIANTS[variant] + ["-o", so, os.path.join(HOSTEMU, "hostemu.cpp")])
    lib = ctypes.CDLL(so)
    if variant == "trace":
        lib.he_trace_read.restype = ctypes.c_size_t
    return lib


def limbs(vals):
    """Python ints -> (n, 8) uint32 limbs (the in-memory layout of Fp256; the same bytes as (n, 4) uint64)"""
    return np.array([_limbs32(v) for v in vals], dtype=np.uint32).reshape(-1, 8)


def ints(arr):
    arr = np.ascontiguousarray(arr).view(np.uint32).reshape(-1, 8)
    return [sum(int(r[j]) << (32 * j) for j in range(8)) for r in arr]


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def run_host(lib, field, prim, tuples):
    """the primitive through a hostemu library -> (n, 8) uint32 result limbs"""
    cols = [limbs([t[i] for t in tuples]) for i in range(ARITY[prim])]
    out = np.empty((len(tuples), 8), dtype=np.uint32)
    n = ctypes.c_size_t(len(tuples))
    if prim == "mul_sub_mul":
        lib.he_field_mul_sub_mul(FIELD_CODE[field], *[_p(c) for c in cols], _p(out), n)
    else:
        b = cols[1] if len(cols) > 1 else np.zeros_like(cols[0])
        lib.he_field_op(FIELD_CODE[field], OPS[prim], _p(cols[0]), _p(b), _p(out), n)
    return out


def read_trace(lib):
    """-> {(file basename, line, instance, instruction): seen bits} of the trace build since the last reset"""
    cap = 8192
    files, lines, seqs = (ctypes.c_char_p * cap)(), (ctypes.c_int32 * cap)(), (ctypes.c_int32 * cap)()
    ops, seen = (ctypes.c_char_p * cap)(), (ctypes.c_uint32 * cap)()
    n = lib.he_trace_read(files, lines, seqs, ops, seen, ctypes.c_size_t(cap))
    out = {}
    for i in range(n):
        key = (os.path.basename(files[i].decode()), lines[i], seqs[i], ops[i].decode())
        out[key] = out.get(key, 0) | seen[i]
    return out


def by_line(trace):
    """instances folded into their call site: {(file basename, line, instruction): seen bits}"""
    out = {}
    for (f, line, _, op), bits in trace.items():
        out[(f, line, op)] = out.get((f, line, op), 0) | bits
    return out


def trace_of(lib, field, prim, tuples):
    lib.he_trace_reset()
    if tuples:
        run_host(lib, field, prim, tuples)
    return read_trace(lib)


def _features(trace):
    return {(k, bit) for k, bits in trace.items() for bit in (1, 2, 4, 8) if bits & bit}


def select(lib, field, prim, fams, chunk=256):
    """greedy, in family order: keep each candidate that shows an (instance, bit) the kept ones have not shown; a chunk
    that adds nothing as a whole is passed over in one call"""
    have, kept = set(), []
    for _, cands in fams:
        for lo in range(0, len(cands), chunk):
            part = cands[lo:lo + chunk]
            if _features(trace_of(lib, field, prim, part)) <= have:
                continue
            for t in part:
                f = _features(trace_of(lib, field, prim, [t]))
                if not f <= have:
                    have |= f; kept.append(t)
    return kept


@functools.lru_cache(maxsize=None)
def _corpus(out_dir, field, prim):
    return tuple(select(build_hostemu(out_dir, "trace"), field, prim, families(field, prim)))


def corpus(out_dir, field, prim):
    """the greedy-selected operand tuples of one primitive over one field (the trace library is built in out_dir)"""
    return list(_corpus(str(out_dir), field, prim))
