"""Poseidon over BN254's Fr and the Poseidon proof transcript -- host-side mirror of what snark-verifier's
`PoseidonTranscript<NativeLoader, _>` does for the INNER snark of both Spectre pipelines (`gen_snark_shplonk`,
lightclient-circuits/src/util/circuit.rs:163-180; reached from prover/src/rpc.rs:144-149). The outer (EVM) proof uses the
Keccak transcript in transcript.py. Like that one, this is the caller's side of the C ABI: it hashes a few hundred field
elements per proof and is nowhere near the GPU hot path.

Two layers, with different pinning:

* The PERMUTATION and its parameters are pinned. `grain_parameters` restates the published parameter generation of the
  Poseidon reference implementation (Grain LFSR in self-shrinking mode: 80-bit state = field type 1 | s-box 0 | field bits | t |
  R_F | R_P | 30 ones, 160 discarded bits, round constants by rejection sampling of `field_bits`-bit integers, then a Cauchy
  matrix 1 / (x_i + y_j) from 2t further draws reduced mod r) -- the same procedure the `poseidon` crates behind halo2-base /
  snark-verifier run ([UPSTREAM] halo2-base `poseidon::hasher::spec::OptimizedPoseidonSpec::new::<R_F, R_P, 0>`, used by the
  reference at lightclient-circuits/src/poseidon.rs:83 and, with T = 3, RATE = 2, R_F = 8, R_P = 57, by the transcript). The
  optimised spec those crates derive is an equivalent re-association of the same permutation. `tests/test_poseidon.py` checks
  the t = 3 instance against the known-answer vector published with the reference implementation (`poseidonperm_x5_254_3`:
  input (0, 1, 2)).
* The SPONGE and the TRANSCRIPT framing are restated from upstream as remembered and are **unpinned**: the reference tree
  holds no Poseidon digest of data that is also in the tree (`.env.example`'s INITIAL_COMMITTEE_POSEIDON is the hash of a
  committee absent from test_data/), and no inner-snark proof. What is restated: state = (2^64, 0, 0); `update` buffers;
  `squeeze` absorbs the buffer RATE elements at a time (a short last chunk is padded with a single 1 right after it; an
  exactly-full buffer is followed by one more permutation of the empty chunk) and returns state[1]; the transcript feeds
  every challenge back in, absorbs a G1 point as (x mod r, y mod r), and writes points compressed (32-byte little-endian x
  with the parity of y in the top bit) and scalars as 32-byte little-endian canonical values. A Rust host keeps
  snark-verifier's own transcript (INTEGRATION.md); this module exists so that the in-repo drivers can run the same protocol
  over either transcript, and is self-consistent with tests/plonk_verifier.py.
"""
from .halo2 import P_MOD, R_MOD, g1_on_curve


def _grain_bits(field_bits, t, r_f, r_p):
    """The self-shrinking Grain LFSR of the Poseidon parameter generation: yields the output bit stream."""
    bits = [int(b) for b in format(1, "02b") + format(0, "04b") + format(field_bits, "012b") + format(t, "012b")
            + format(r_f, "010b") + format(r_p, "010b") + "1" * 30]

    def step():
        b = bits[62] ^ bits[51] ^ bits[38] ^ bits[23] ^ bits[13] ^ bits[0]
        bits.pop(0); bits.append(b)
        return b
    for _ in range(160):
        step()
    while True:
        b = step()
        while b == 0:           # a 0 discards the bit after it
            step(); b = step()
        yield step()


def grain_parameters(t, r_f, r_p, field_bits=254, modulus=R_MOD):
    """-> (round constants [(r_f + r_p)][t], mds [t][t]) as integers."""
    stream = _grain_bits(field_bits, t, r_f, r_p)

    def draw():
        v = 0
        for _ in range(field_bits):
            v = (v << 1) | next(stream)
        return v
    constants = []
    for _ in range(r_f + r_p):
        row = []
        for _ in range(t):
            v = draw()
            while v >= modulus:
                v = draw()
            row.append(v)
        constants.append(row)
    while True:
        xy = [draw() % modulus for _ in range(2 * t)]
        xs, ys = xy[:t], xy[t:]
        if len(set(xy)) == 2 * t and all((x + y) % modulus for x in xs for y in ys):
            break
    mds = [[pow((xs[i] + ys[j]) % modulus, modulus - 2, modulus) for j in range(t)] for i in range(t)]
    return constants, mds


class Spec:
    """Poseidon parameters for width t (x^5 s-box): r_f full rounds split evenly around r_p partial rounds."""
    _cache = {}

    def __new__(cls, t, r_f, r_p):
        key = (t, r_f, r_p)
        if key not in cls._cache:
            self = super().__new__(cls)
            self.t, self.r_f, self.r_p = t, r_f, r_p
            self.constants, self.mds = grain_parameters(t, r_f, r_p)
            cls._cache[key] = self
        return cls._cache[key]

    def permute(self, state):
        t, m = self.t, self.mds
        state = list(state)
        half = self.r_f // 2
        for rnd in range(self.r_f + self.r_p):
            state = [(s + c) % R_MOD for s, c in zip(state, self.constants[rnd])]
            if rnd < half or rnd >= half + self.r_p:
                state = [pow(s, 5, R_MOD) for s in state]
            else:
                state[0] = pow(state[0], 5, R_MOD)
            state = [sum(m[i][j] * state[j] for j in range(t)) % R_MOD for i in range(t)]
        return state


class Poseidon:
    """The sponge as snark-verifier's `util::hash::Poseidon` drives it (restated, unpinned -- module docstring)."""

    def __init__(self, t=3, rate=2, r_f=8, r_p=57):
        assert rate == t - 1
        self.spec, self.rate = Spec(t, r_f, r_p), rate
        self.state = [1 << 64] + [0] * (t - 1)
        self.buf = []

    def update(self, elements):
        self.buf.extend(int(e) % R_MOD for e in elements)

    def _absorb(self, chunk):
        s = list(self.state)
        for i, v in enumerate(chunk):
            s[1 + i] = (s[1 + i] + v) % R_MOD
        if len(chunk) < self.rate:
            s[1 + len(chunk)] = (s[1 + len(chunk)] + 1) % R_MOD
        self.state = self.spec.permute(s)

    def squeeze(self):
        buf, self.buf = self.buf, []
        for i in range(0, len(buf), self.rate):
            self._absorb(buf[i:i + self.rate])
        if len(buf) % self.rate == 0:
            self._absorb([])
        return self.state[1]


def compress_g1(xy):
    """32-byte little-endian x with the parity of y in the top bit (the identity is all zero)."""
    x, y = xy
    if x == 0 and y == 0:
        return bytes(32)
    b = bytearray(int(x).to_bytes(32, "little"))
    b[31] |= (int(y) & 1) << 7
    return bytes(b)


def decompress_g1(b):
    b = bytearray(b)
    if not any(b):
        return (0, 0)
    odd = b[31] >> 7
    b[31] &= 0x7f
    x = int.from_bytes(b, "little")
    if x >= P_MOD:
        raise ValueError("non-canonical x coordinate in proof")
    y = pow((x * x * x + 3) % P_MOD, (P_MOD + 1) // 4, P_MOD)          # p = 3 mod 4
    if not g1_on_curve(x, y):
        raise ValueError("proof point is not on the curve")
    return (x, y if (y & 1) == odd else P_MOD - y)


class PoseidonTranscriptWrite:
    """Prover side, same interface as transcript.EvmTranscriptWrite (create_proof takes either)."""

    def __init__(self, vk_digest, t=3, rate=2, r_f=8, r_p=57):
        self.hasher = Poseidon(t, rate, r_f, r_p)
        self.proof = bytearray()
        self.common_scalar(vk_digest)            # VerifyingKey::hash_into

    def common_scalar(self, v):
        self.hasher.update([int(v) % R_MOD])

    def common_ec_point(self, xy):
        x, y = xy
        if x == 0 and y == 0:
            raise ValueError("PoseidonTranscript cannot absorb the point at infinity")
        self.hasher.update([int(x) % R_MOD, int(y) % R_MOD])

    def write_scalar(self, v):
        self.common_scalar(v)
        self.proof += (int(v) % R_MOD).to_bytes(32, "little")

    def write_ec_point(self, xy):
        self.common_ec_point(xy)
        self.proof += compress_g1(xy)

    def squeeze_challenge(self):
        c = self.hasher.squeeze()
        self.hasher.update([c])
        return c


class PoseidonTranscriptRead(PoseidonTranscriptWrite):
    """Verifier side over a proof byte string."""

    def __init__(self, vk_digest, proof, **kw):
        super().__init__(vk_digest, **kw)
        self.stream, self.pos = bytes(proof), 0

    def read_scalar(self):
        v = int.from_bytes(self.stream[self.pos:self.pos + 32], "little"); self.pos += 32
        if v >= R_MOD:
            raise ValueError("non-canonical scalar in proof")
        self.common_scalar(v)
        return v

    def read_ec_point(self):
        xy = decompress_g1(self.stream[self.pos:self.pos + 32]); self.pos += 32
        self.common_ec_point(xy)
        return xy
