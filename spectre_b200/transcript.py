"""EVM (Keccak-256) proof transcript -- host-side mirror of snark-verifier's `EvmTranscript`
([UPSTREAM] snark-verifier/src/system/halo2/transcript/evm.rs), the transcript Spectre's `gen_evm_proof_shplonk`
uses (lightclient-circuits/src/util/circuit.rs:196-218). Its byte conventions are pinned by the reference's committed
verifier contracts, which replay it in Yul (contracts/snark-verifiers/sync_step_verifier.sol:41-56,78,84-85,...):

  * state = a byte buffer, initially the 32-byte verifying-key digest;
  * common_scalar appends the 32-byte big-endian canonical value; common_ec_point appends x then y the same way;
  * squeeze_challenge hashes the buffer (with one extra byte 0x01 when the buffer is exactly 32 bytes long, i.e. two
    squeezes in a row), keeps the 32-byte digest as the new buffer and returns digest mod r;
  * the proof stream holds exactly the written points (64 B) and scalars (32 B), big-endian.

The transcript is the caller's side of the C ABI (it orders the calls and owns the challenges); nothing here is on
the GPU hot path. hashlib has SHA-3 but not the original Keccak padding, so Keccak-f[1600] is spelled out below.
"""
from .halo2 import R_MOD, g1_on_curve

_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M64 = (1 << 64) - 1


def _rol(v, n):
    n %= 64
    return ((v << n) | (v >> (64 - n))) & _M64 if n else v


def _keccak_f(a):
    for rc in _RC:
        c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rol(c[(x + 1) % 5], 1) for x in range(5)]
        a = [[a[x][y] ^ d[x] for y in range(5)] for x in range(5)]
        b = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                b[y][(2 * x + 3 * y) % 5] = _rol(a[x][y], _ROT[x][y])
        a = [[b[x][y] ^ ((~b[(x + 1) % 5][y]) & b[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        a[0][0] ^= rc
    return a


def keccak256(data):
    """Keccak-256 with the original 0x01 domain padding (what the EVM's KECCAK256 opcode computes)."""
    rate = 136
    msg = bytearray(data)
    msg.append(0x01)
    while len(msg) % rate:
        msg.append(0)
    msg[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(msg), rate):
        for i in range(rate // 8):
            a[i % 5][i // 5] ^= int.from_bytes(msg[off + 8 * i: off + 8 * i + 8], "little")
        a = _keccak_f(a)
    return b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))


class EvmTranscriptWrite:
    """Prover side: write_* both absorb and append to the proof stream; common_* only absorb."""

    def __init__(self, vk_digest):
        self.buf = bytearray(int(vk_digest).to_bytes(32, "big"))
        self.proof = bytearray()
        self.absorbed = []          # byte length of every hashed buffer, for layout checks against the verifier contract

    def common_scalar(self, v):
        self.buf += int(v % R_MOD).to_bytes(32, "big")

    def common_ec_point(self, xy):
        x, y = xy
        if x == 0 and y == 0:
            raise ValueError("EvmTranscript cannot absorb the point at infinity")   # upstream: Error::Transcript
        self.buf += int(x).to_bytes(32, "big") + int(y).to_bytes(32, "big")

    def write_scalar(self, v):
        self.common_scalar(v)
        self.proof += int(v % R_MOD).to_bytes(32, "big")

    def write_ec_point(self, xy):
        self.common_ec_point(xy)
        self.proof += int(xy[0]).to_bytes(32, "big") + int(xy[1]).to_bytes(32, "big")

    def squeeze_challenge(self):
        data = bytes(self.buf) + (b"\x01" if len(self.buf) == 32 else b"")
        self.absorbed.append(len(data))
        h = keccak256(data)
        self.buf = bytearray(h)
        return int.from_bytes(h, "big") % R_MOD


class EvmTranscriptRead(EvmTranscriptWrite):
    """Verifier side over a proof byte string."""

    def __init__(self, vk_digest, proof):
        super().__init__(vk_digest)
        self.stream = bytes(proof)
        self.pos = 0

    def read_scalar(self):
        v = int.from_bytes(self.stream[self.pos:self.pos + 32], "big"); self.pos += 32
        if v >= R_MOD:
            raise ValueError("non-canonical scalar in proof")
        self.common_scalar(v)
        return v

    def read_ec_point(self):
        x = int.from_bytes(self.stream[self.pos:self.pos + 32], "big"); y = int.from_bytes(self.stream[self.pos + 32:self.pos + 64], "big"); self.pos += 64
        if not g1_on_curve(x, y):
            raise ValueError("proof point is not on the curve")
        self.common_ec_point((x, y))
        return (x, y)
