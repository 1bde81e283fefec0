"""A pure-Python BN254 optimal ate pairing -- TEST INFRASTRUCTURE, the independent reference for csrc/pairing.cuh.

Tower (halo2curves' bn256): Fq2 = Fq[u]/(u^2 + 1), Fq6 = Fq2[v]/(v^3 - xi) with xi = 9 + u, Fq12 = Fq6[w]/(w^2 - v).
Elements are nested tuples of canonical ints: Fq2 (c0, c1), Fq6 (c0, c1, c2), Fq12 (c0, c1).

It shares nothing with the device code but the tower. The Miller loop runs on Q untwisted into E(Fq12) (x' w^2, y' w^3) with
affine chord-and-tangent arithmetic over Fq12 and the plain binary digits of 6u + 2; pi(Q) and pi^2(Q) are the coordinates
raised to p and p^2; Frobenius maps are powers; the final exponentiation is one power by the literal (p^12 - 1) / r. Vertical
lines are left out: their values lie in Fq6, which the final exponentiation sends to one.
"""
from tests import pyref

P = pyref.P_MOD
R = pyref.R_MOD
U = 4965661367192848881
ATE_LOOP = 6 * U + 2
FINAL_EXP = (P ** 12 - 1) // R

# the generator of G2 (halo2curves' G2Affine::generator, EIP-197): x = x.c0 + x.c1 u, y likewise
G2_GEN = ((0x1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed, 0x198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2),
          (0x12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa, 0x090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b))
G1_GEN = (1, 2)


# ---- Fq2 -------------------------------------------------------------------------------------------------------------
F2_ZERO, F2_ONE = (0, 0), (1, 0)
XI = (9, 1)


def f2_add(a, b): return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)
def f2_sub(a, b): return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)
def f2_neg(a): return (-a[0] % P, -a[1] % P)
def f2_mul(a, b): return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)
def f2_scale(a, s): return (a[0] * s % P, a[1] * s % P)
def f2_conj(a): return (a[0], -a[1] % P)


def f2_inv(a):
    d = pow(a[0] * a[0] + a[1] * a[1], -1, P)
    return (a[0] * d % P, -a[1] * d % P)


def f2_pow(a, e):
    r = F2_ONE
    while e:
        if e & 1:
            r = f2_mul(r, a)
        a = f2_mul(a, a)
        e >>= 1
    return r


def f2_sqrt(a):
    """a square root of a in Fq2, or None (p = 3 mod 4: Adj and Rodriguez-Henriquez, Algorithm 9)"""
    a1 = f2_pow(a, (P - 3) // 4)
    alpha = f2_mul(f2_mul(a1, a1), a)
    x0 = f2_mul(a1, a)
    if alpha == (P - 1, 0):
        x = f2_mul((0, 1), x0)
    else:
        x = f2_mul(f2_pow(f2_add(F2_ONE, alpha), (P - 1) // 2), x0)
    return x if f2_mul(x, x) == (a[0] % P, a[1] % P) else None


# ---- Fq6, Fq12: schoolbook products reduced by v^3 = xi and w^2 = v --------------------------------------------------
F6_ZERO = (F2_ZERO, F2_ZERO, F2_ZERO)
F6_ONE = (F2_ONE, F2_ZERO, F2_ZERO)
F12_ONE = (F6_ONE, F6_ZERO)


def f6_add(a, b): return tuple(f2_add(x, y) for x, y in zip(a, b))
def f6_sub(a, b): return tuple(f2_sub(x, y) for x, y in zip(a, b))
def f6_neg(a): return tuple(f2_neg(x) for x in a)


def f6_mul(a, b):
    t = [F2_ZERO] * 5
    for i in range(3):
        for j in range(3):
            t[i + j] = f2_add(t[i + j], f2_mul(a[i], b[j]))
    return (f2_add(t[0], f2_mul(XI, t[3])), f2_add(t[1], f2_mul(XI, t[4])), t[2])


def f6_mul_v(a): return (f2_mul(XI, a[2]), a[0], a[1])


def f6_inv(a):
    """a^-1 = a^(p^2) a^(p^4) / N(a), N(a) = a a^(p^2) a^(p^4) in Fq2; a^(p^2k) maps c_j v^j to c_j xi^(j (p^2k - 1) / 3) v^j"""
    def frob2(x, k):
        return tuple(f2_mul(c, _XI_POW[k][j]) for j, c in enumerate(x))
    conj = f6_mul(frob2(a, 1), frob2(a, 2))
    norm = f6_mul(a, conj)
    assert norm[1] == F2_ZERO and norm[2] == F2_ZERO
    ni = f2_inv(norm[0])
    return tuple(f2_mul(c, ni) for c in conj)


_XI_POW = {k: [f2_pow(XI, j * (P ** (2 * k) - 1) // 3) for j in range(3)] for k in (1, 2)}


def f12_mul(a, b):
    return (f6_add(f6_mul(a[0], b[0]), f6_mul_v(f6_mul(a[1], b[1]))), f6_add(f6_mul(a[0], b[1]), f6_mul(a[1], b[0])))


def f12_sqr(a): return f12_mul(a, a)
def f12_conj(a): return (a[0], f6_neg(a[1]))


def f12_inv(a):
    """(a0 + a1 w)^-1 = (a0 - a1 w) / (a0^2 - v a1^2)"""
    d = f6_inv(f6_sub(f6_mul(a[0], a[0]), f6_mul_v(f6_mul(a[1], a[1]))))
    return (f6_mul(a[0], d), f6_neg(f6_mul(a[1], d)))


def f12_pow(a, e):
    r = F12_ONE
    for bit in bin(e)[2:]:
        r = f12_sqr(r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def f12_frobenius(a, k):
    """a^(p^k)"""
    return f12_pow(a, P ** k)


def f12_from_fq(x): return (((x % P, 0), F2_ZERO, F2_ZERO), F6_ZERO)
def f12_add(a, b): return (f6_add(a[0], b[0]), f6_add(a[1], b[1]))
def f12_sub(a, b): return (f6_sub(a[0], b[0]), f6_sub(a[1], b[1]))


# ---- G2 on the twist y^2 = x^3 + 3 / xi over Fq2 (affine; None = identity) ------------------------------------------
B_TWIST = f2_mul((3, 0), f2_inv(XI))


def g2_on_curve(q):
    return q is None or f2_sub(f2_mul(q[1], q[1]), f2_add(f2_mul(f2_mul(q[0], q[0]), q[0]), B_TWIST)) == F2_ZERO


def g2_neg(q): return None if q is None else (q[0], f2_neg(q[1]))


def g2_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    if a[0] == b[0]:
        if f2_add(a[1], b[1]) == F2_ZERO:
            return None
        lam = f2_mul(f2_scale(f2_mul(a[0], a[0]), 3), f2_inv(f2_scale(a[1], 2)))
    else:
        lam = f2_mul(f2_sub(b[1], a[1]), f2_inv(f2_sub(b[0], a[0])))
    x3 = f2_sub(f2_sub(f2_mul(lam, lam), a[0]), b[0])
    return (x3, f2_sub(f2_mul(lam, f2_sub(a[0], x3)), a[1]))


def g2_mul(q, k):
    r = None
    while k:
        if k & 1:
            r = g2_add(r, q)
        q = g2_add(q, q)
        k >>= 1
    return r


def g2_twist_point_outside_subgroup(start=1):
    """the first twist point (x, y) with x = start, start + 1, ... (real x) whose [r] multiple is not the identity; no cofactor is
    cleared, so its order has a factor of the cofactor 2p - r"""
    x = start
    while True:
        y = f2_sqrt(f2_add(f2_mul(f2_mul((x, 0), (x, 0)), (x, 0)), B_TWIST))
        if y is not None and g2_mul(((x, 0), y), R) is not None:
            return ((x, 0), y)
        x += 1


# ---- pairing ---------------------------------------------------------------------------------------------------------
def _untwist(q):
    """(x', y') on the twist -> (x' w^2, y' w^3) in E(Fq12): w^2 = v, w^3 = v w"""
    return ((F2_ZERO, q[0], F2_ZERO), F6_ZERO), (F6_ZERO, (F2_ZERO, q[1], F2_ZERO))


def _line(t, slope, p):
    """the line through t with this slope, at the Fq12 point p: y_p - y_t - slope (x_p - x_t)"""
    return f12_sub(f12_sub(p[1], t[1]), f12_mul(slope, f12_sub(p[0], t[0])))


def _add(t, q):
    """t + q in E(Fq12) (neither the identity, t != -q) and the slope of the chord / tangent"""
    if t == q:
        slope = f12_mul(f12_mul(f12_from_fq(3), f12_sqr(t[0])), f12_inv(f12_add(t[1], t[1])))
    else:
        slope = f12_mul(f12_sub(q[1], t[1]), f12_inv(f12_sub(q[0], t[0])))
    x3 = f12_sub(f12_sub(f12_sqr(slope), t[0]), q[0])
    return (x3, f12_sub(f12_mul(slope, f12_sub(t[0], x3)), t[1])), slope


def miller_loop(p, q):
    """f_{6u+2,Q}(P) l_{[6u+2]Q, pi(Q)}(P) l_{[6u+2]Q + pi(Q), -pi^2(Q)}(P), up to factors in Fq6; 1 if either point is the identity.
    p: (x, y) ints or None; q: ((x.c0, x.c1), (y.c0, y.c1)) or None."""
    if p is None or q is None:
        return F12_ONE
    pp = (f12_from_fq(p[0]), f12_from_fq(p[1]))
    qq = _untwist(q)
    f, t = F12_ONE, qq
    for bit in bin(ATE_LOOP)[3:]:
        t2, slope = _add(t, t)
        f = f12_mul(f12_sqr(f), _line(t, slope, pp))
        t = t2
        if bit == "1":
            t2, slope = _add(t, qq)
            f = f12_mul(f, _line(t, slope, pp))
            t = t2
    q1 = (f12_frobenius(qq[0], 1), f12_frobenius(qq[1], 1))
    q2 = (f12_frobenius(qq[0], 2), f12_frobenius(qq[1], 2))
    q2 = (q2[0], f12_sub(f12_from_fq(0), q2[1]))
    t2, slope = _add(t, q1)
    f = f12_mul(f, _line(t, slope, pp))
    _, slope = _add(t2, q2)
    return f12_mul(f, _line(t2, slope, pp))


def final_exponentiation(f):
    return f12_pow(f, FINAL_EXP)


def pairing(p, q):
    return final_exponentiation(miller_loop(p, q))


def multi_pairing(ps, qs):
    """prod_i e(ps[i], qs[i]) with one final exponentiation"""
    f = F12_ONE
    for p, q in zip(ps, qs):
        f = f12_mul(f, miller_loop(p, q))
    return final_exponentiation(f)


def pairing_check(ps, qs):
    return multi_pairing(ps, qs) == F12_ONE


# ---- layouts: Gt as 12 Fq values in halo2curves' order c0.c0.c0 ... c1.c2.c1 ----------------------------------------
def f12_flat(a):
    return [c for f6 in a for f2 in f6 for c in f2]


def f12_unflat(v):
    v = [int(x) % P for x in v]
    f2 = [(v[2 * i], v[2 * i + 1]) for i in range(6)]
    return ((f2[0], f2[1], f2[2]), (f2[3], f2[4], f2[5]))


def f6_flat(a):
    return [c for f2 in a for c in f2]


def f6_unflat(v):
    v = [int(x) % P for x in v]
    return ((v[0], v[1]), (v[2], v[3]), (v[4], v[5]))


# ---- the library's in-memory layouts: Montgomery limbs, 4 x u64 per Fq ----------------------------------------------
_MONT = (1 << 256) % P
_MONT_INV = pow(_MONT, -1, P)
_M64 = (1 << 64) - 1


def fq_limbs(vals):
    """canonical ints -> (len, 4) uint64 Montgomery limbs"""
    import numpy as np
    return np.array([[(v % P * _MONT % P >> (64 * j)) & _M64 for j in range(4)] for v in vals], dtype=np.uint64).reshape(-1, 4)


def fq_ints(arr):
    """Montgomery limbs (..., 4) -> canonical ints"""
    import numpy as np
    arr = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 4)
    return [(int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192) * _MONT_INV % P for r in arr]


def g1_limbs(p):
    """G1 affine (x, y) or None -> (8,) uint64, identity (0, 0)"""
    return fq_limbs([0, 0] if p is None else list(p)).reshape(8)


def g2_limbs(q):
    """G2 affine ((x.c0, x.c1), (y.c0, y.c1)) or None -> (16,) uint64 in the params file's order x.c0, x.c1, y.c0, y.c1"""
    return fq_limbs([0, 0, 0, 0] if q is None else [q[0][0], q[0][1], q[1][0], q[1][1]]).reshape(16)


def g2_from_limbs(a):
    v = fq_ints(a)
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


def gt_from_limbs(a):
    return f12_unflat(fq_ints(a))


def gt_limbs(f):
    return fq_limbs(f12_flat(f))
