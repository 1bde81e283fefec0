"""The MSM at every geometry it can choose, against the O(n) known-secret commitment of the seed-0 SRS.

msm_choose_c picks the window width c from the length (without window tables) or from the basis length (with them), and c
fixes the number of windows W, of buckets B = 2^(c-1), and the bucket-reduction shape (msm_tail_shape: row / column blocks
nbr x nbc of msm_weighted_kernel and the host fold msm_tail_finish). The chunk length comes from n * W on the host and is
cut back on the device when the sorted list is short (msm_effective_chunk), and bucket chains of more than 24 / 4096 chunk
pieces go to the giant / huge kernels. The widths are derived here from the library itself (spb_msm_geometry, binary search
over 1 <= n <= 2^24), so a new choice of widths widens these tests by itself.

Every result is compared with commit(a) = (sum_i a_i tau^i) * G (orc.commit_known_tau), which uses no MSM code. Where the
number of sorted entries M is known in advance (columns of ones, of small values, of chosen digits), spb_last_msm_adds
= M + 2 * BW * B proves which geometry ran: BW = W bucket sets without tables, 1 with them."""
import gc

import numpy as np
import pytest

from tests import pyref
from tests.gpu_common import be  # noqa: F401

pytestmark = pytest.mark.gpu

R = pyref.R_MOD
NMAX = 1 << 24
K23 = 23
LONG_CHUNK_MIN_ENTRIES = 1 << 23   # msm.cuh kLongChunkMinEntries: the long chunk (96) only from this many sorted entries on
LONG_CHUNK, SHORT_CHUNK = 96, 32
STITCH_CAP, HUGE_CHAIN, GIANT_BLOCKS = 24, 4096, 256


def _release(be):
    import torch
    gc.collect()
    torch.cuda.synchronize()
    be.release_workspace()
    torch.cuda.empty_cache()


def _tail_shape(c):
    """msm_tail_shape: (m_log, R, C, nbr, nbc)"""
    bits = c - 1
    m_log = min(bits, 3)
    bits -= m_log
    c_log = bits // 2
    r_log = bits - c_log
    return m_log, 1 << r_log, 1 << c_log, ((1 << r_log) + 127) // 128, ((1 << c_log) + 127) // 128


def _width_ranges(be, tables):
    """[(c, W, n_lo, n_hi)] over 1 <= n <= 2^24: the last n of each width by binary search (the width never decreases with n)"""
    out, n = [], 1
    while n <= NMAX:
        c, W = be.msm_geometry(n, tables)
        lo, hi = n, NMAX
        while lo < hi:
            mid = (lo + hi + 1) // 2
            if be.msm_geometry(mid, tables)[0] == c:
                lo = mid
            else:
                hi = mid - 1
        out.append((c, W, n, lo))
        n = lo + 1
    return out


def _tabled_geometry(be, n, bases):
    """(c, W, BW) of an MSM of n scalars on a handle of n points per basis after precompute(): spb_srs_precompute builds the
    tables only while W x n points x 64 B x the resident bases fit a quarter of the device's memory; otherwise the handle keeps
    the plain layout and the width of n scalars without tables"""
    import torch
    c, W = be.msm_geometry(n, True)
    if W * n * 64 * bases > torch.cuda.get_device_properties(0).total_memory // 4:
        c, W = be.msm_geometry(n, False)
        return c, W, W
    return c, W, 1


def _host_chunk(est_entries, sm_count):
    """choose_chunk (msm.cu): the chunk length the host asks for, from the upper bound n * W on the entries"""
    if est_entries >= LONG_CHUNK_MIN_ENTRIES:
        return LONG_CHUNK
    wave = sm_count * 512.0
    waves = est_entries / 32.0 / wave
    if waves < 1.0:
        return 32
    w = 1.0 if waves < 1.5 else float(int(waves + 0.5))
    return min(48, max(24, int(est_entries / (w * wave)) + 1))


def _signed_digits(s, c, W):
    """number of non-zero signed c-bit digits of s, as msm.cuh's DigitIter makes them: raw = window + carry, and a raw above
    B = 2^(c-1) becomes raw - 2^c with a carry into the next window"""
    B, full, mask, carry, count = 1 << (c - 1), 1 << c, (1 << c) - 1, 0, 0
    for w in range(W):
        raw = ((s >> (c * w)) & mask) + carry
        carry = 1 if raw > B else 0
        count += (raw - full if carry else raw) != 0
    assert carry == 0, "a carry out of the top window: W * c leaves no spare bit"
    return count


def _mont(be, orc, canon):
    """canonical limbs (n, 4), each value below r -> Montgomery limbs, by one device product with R^2 mod r"""
    return be.vec_scale(canon, orc.fr([(1 << 256) % R])[0])


def _small_values(be, orc, vals):
    canon = np.zeros((len(vals), 4), dtype=np.uint64)
    canon[:, 0] = vals
    return _mont(be, orc, canon)


def _witness_canon(n, rng):
    """witness-like: 70% zero, 20% below 2^16, 9% below 2^104, 1% below 2^253"""
    u = rng.random(n)
    canon = np.zeros((n, 4), dtype=np.uint64)
    small, mid, big = (u >= 0.7) & (u < 0.9), (u >= 0.9) & (u < 0.99), u >= 0.99
    canon[small, 0] = rng.integers(0, 1 << 16, int(small.sum()), dtype=np.uint64)
    canon[mid, 0] = rng.integers(0, 1 << 64, int(mid.sum()), dtype=np.uint64, endpoint=False)
    canon[mid, 1] = rng.integers(0, 1 << 40, int(mid.sum()), dtype=np.uint64)
    canon[big, :3] = rng.integers(0, 1 << 64, (int(big.sum()), 3), dtype=np.uint64, endpoint=False)
    canon[big, 3] = rng.integers(0, 1 << 61, int(big.sum()), dtype=np.uint64)
    return canon


def _boundary_scalars(c, W, count, rng):
    """scalars sum_j v_j 2^(c j) with every window value v_j in {0, B, B + 1, 2^c - 1} (a digit of exactly +B, the largest
    bucket key; a carry; a carry chain), the highest windows cleared until the value is below r"""
    B = 1 << (c - 1)
    choice = (0, B, B + 1, (1 << c) - 1)
    out = []
    for picks in rng.integers(0, 4, (count, W)):
        v = [choice[p] for p in picks]
        top = W
        while sum(d << (c * j) for j, d in enumerate(v[:top])) >= R:
            top -= 1
        out.append(sum(d << (c * j) for j, d in enumerate(v[:top])))
    return out


def _same_digit_scalar(c, W):
    """every window holds the digit +B (the largest bucket key) as far as the value stays below r: -> (scalar, windows)"""
    B, top = 1 << (c - 1), W
    while sum(B << (c * j) for j in range(top)) >= R:
        top -= 1
    return sum(B << (c * j) for j in range(top)), top


class Columns:
    """Scalar columns of 2^24 Montgomery elements shared by the tests (they take prefixes), and the known-secret commitment of
    each prefix, computed once"""

    def __init__(self, be, orc):
        self.be, self.orc, self._cols, self._known = be, orc, {}, {}

    def __getitem__(self, name):
        if name not in self._cols:
            be, orc = self.be, self.orc
            if name == "uniform":
                col = orc.fr_random_chacha(NMAX, 0x6e0a)
            elif name == "ones":
                col = np.repeat(orc.fr([1]), NMAX, axis=0)
            elif name == "minus_one":
                col = np.repeat(orc.fr([R - 1]), NMAX, axis=0)
            elif name == "witness":
                col = _mont(be, orc, _witness_canon(NMAX, np.random.default_rng(0x6e0b)))
            else:
                raise KeyError(name)
            self._cols[name] = col
        return self._cols[name]

    def known(self, name, n):
        if (name, n) not in self._known:
            self._known[(name, n)] = self.orc.commit_known_tau(self[name][:n])
        return self._known[(name, n)]


class _Held:
    """An SRS handle a class of tests shares; its teardown drops the handle (and the device memory) before the next class"""

    def __init__(self, params):
        self.params, self._g = params, None

    def g(self):
        """the monomial basis, downloaded once"""
        if self._g is None:
            self._g = self.params.get_g(0, self.params.n)
        return self._g


@pytest.fixture(scope="module")
def cols(be, orc):
    return Columns(be, orc)


@pytest.fixture(scope="module")
def geometries(be):
    table = {tables: _width_ranges(be, tables) for tables in (False, True)}
    print("\nMSM geometries for 1 <= n <= 2^24 (n: the scalar count without tables, the basis length with them)")
    print("%3s %6s %10s %10s %3s %6s %4s %4s %3s %3s" % ("c", "tables", "n_lo", "n_hi", "W", "m_log", "R", "C", "nbr", "nbc"))
    for tables, rows in table.items():
        for c, W, lo, hi in rows:
            print("%3d %6s %10d %10d %3d %6d %4d %4d %3d %3d" % ((c, "yes" if tables else "no", lo, hi, W) + _tail_shape(c)))
    return table


def _check(failures, orc, what, got, want, be=None, adds=None):
    if not np.array_equal(orc.g1_to_affine(got), want):
        failures.append("%s: commitment differs from the known-secret value" % what)
    if adds is not None and be.last_msm_adds != adds:
        failures.append("%s: last_msm_adds = %d, expected %d" % (what, be.last_msm_adds, adds))


def test_window_widths_are_derived_from_the_library(be, geometries):
    """The width ranges tile [1, 2^24] without gaps, each width appears once, widths grow with n, W * c >= 255 (a spare bit
    above the 254-bit scalar for the last carry), and lengths between the binary-search points get the width of their range."""
    for tables, rows in geometries.items():
        assert rows[0][2] == 1 and rows[-1][3] == NMAX
        assert all(a[3] + 1 == b[2] for a, b in zip(rows, rows[1:])), rows
        assert all(a[0] < b[0] for a, b in zip(rows, rows[1:])), rows
        for c, W, lo, hi in rows:
            assert W * c >= 255 and (W - 1) * c < 255, (c, W)
        probes = sorted({int(x) for x in np.geomspace(1, NMAX, 3000)} | {r[2] - 1 for r in rows[1:]} | {r[3] + 1 for r in rows[:-1]})
        for n in probes:
            want = next(c for c, W, lo, hi in rows if lo <= n <= hi)
            assert be.msm_geometry(n, tables)[0] == want, (n, tables)


@pytest.fixture(scope="class")
def srs24(be, orc):
    """the seed-0 SRS of 2^24 points, without tables until the last test of its class; workspaces released around it"""
    from spectre_b200.halo2 import ParamsKZG
    _release(be)
    hold = _Held(ParamsKZG.setup(be, 24, orc.srs_tau()))
    yield hold
    hold.params = hold._g = None
    _release(be)


@pytest.fixture(scope="class")
def srs23(be, orc):
    """the seed-0 SRS of 2^23 points with window tables of both bases; workspaces released around it"""
    from spectre_b200.halo2 import ParamsKZG
    _release(be)
    hold = _Held(ParamsKZG.setup(be, K23, orc.srs_tau()).precompute())
    yield hold
    hold.params = hold._g = None
    _release(be)


class TestOnTheK24Srs:
    """One seed-0 SRS of 2^24 points without tables: the plain widths through commit, the tabled ones through handles of
    the first n monomial points with tables, then the K = 24 handle itself after precompute()."""

    def test_plain_widths_at_both_ends(self, be, orc, geometries, cols, srs24):
        """Every plain width at its lowest and highest length, on a uniform column and on ones (M = n); c = 19, the only shape
        with two row blocks and one column block, also on a witness-like and an all-(r - 1) column, and once through
        best_multiexp (spb_msm_raw, the path of the Rust shim)."""
        failures = []
        for c, W, lo, hi in geometries[False]:
            B = 1 << (c - 1)
            names = ("uniform", "ones") + (("witness", "minus_one") if c == 19 else ())
            for n in sorted({lo, hi}):
                for name in names:
                    got = srs24.params.commit(cols[name][:n])
                    M = {"ones": n, "minus_one": n * _signed_digits(R - 1, c, W)}.get(name)
                    _check(failures, orc, "plain c=%d n=%d %s" % (c, n, name), got, cols.known(name, n), be, None if M is None else M + 2 * W * B)
            if c == 19:
                got = be.best_multiexp(cols["uniform"][:lo], srs24.g()[:lo])
                _check(failures, orc, "best_multiexp c=19 n=%d" % lo, got, cols.known("uniform", lo))
        assert not failures, "\n".join(failures)

    def test_tabled_widths_at_both_ends(self, be, orc, geometries, cols, srs24):
        """Every tabled width at the lowest and highest basis length that selects it: from_bases(g[:len]).precompute() and
        multiexp over the whole basis; c = 19 (reachable only through resident bases) also on witness-like and all-(r - 1)."""
        from spectre_b200.halo2 import ParamsKZG
        failures = []
        for c, W, lo, hi in geometries[True]:
            for n in sorted({lo, hi}):
                BW = _tabled_geometry(be, n, 1)[2]
                assert BW == 1, "the tables of %d points do not fit a quarter of the device" % n
                handle = ParamsKZG.from_bases(be, srs24.g()[:n]).precompute()
                for name in ("uniform", "ones") + (("witness", "minus_one") if c == 19 else ()):
                    got = handle.multiexp(cols[name][:n])
                    M = {"ones": n, "minus_one": n * _signed_digits(R - 1, c, W)}.get(name)
                    _check(failures, orc, "tabled c=%d n=%d %s" % (c, n, name), got, cols.known(name, n), be,
                           None if M is None else M + 2 * (1 << (c - 1)))
                del handle
        assert not failures, "\n".join(failures)

    def test_digit_boundary_columns(self, be, orc, geometries, srs24):
        """At every width, plain and tabled, at the highest length that selects it: scalars whose windows are 0, B, B + 1 or
        2^c - 1 (the largest key +B, a carry, a carry chain). M = the number of non-zero signed digits, counted here."""
        from spectre_b200.halo2 import ParamsKZG
        rng = np.random.default_rng(0x6e0c)
        failures = []
        for tables in (False, True):
            for c, W, lo, hi in geometries[tables]:
                n = hi
                P = min(n, 1024)
                pats = _boundary_scalars(c, W, P, rng)
                digits = [_signed_digits(s, c, W) for s in pats]
                col = np.resize(orc.fr(pats), (n, 4))          # pattern i % P at row i
                M = (n // P) * sum(digits) + sum(digits[: n % P])
                want = orc.commit_known_tau(col)
                if tables:
                    handle = ParamsKZG.from_bases(be, srs24.g()[:n]).precompute()
                    got, BW = handle.multiexp(col), _tabled_geometry(be, n, 1)[2]
                    del handle
                else:
                    got, BW = srs24.params.commit(col), W
                _check(failures, orc, "%s c=%d n=%d digit boundaries" % ("tabled" if tables else "plain", c, n), got, want, be, M + 2 * BW * (1 << (c - 1)))
        assert not failures, "\n".join(failures)

    def test_chunk_branches_pinned_by_the_entry_count(self, be, orc, srs24):
        """Small values (one digit each: M = the number of non-zero scalars). Plain 2^23: the host asks for the long chunk, and
        2^23 - 1 entries take the short-chunk fallback on the device while 2^23 keep the long one. Plain 2^18 and tabled 2^19
        land in choose_chunk's 24..48 branch."""
        import torch
        from spectre_b200.halo2 import ParamsKZG
        rng = np.random.default_rng(0x6e0d)
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        failures = []
        n = 1 << 23
        c, W = be.msm_geometry(n, False)
        B = 1 << (c - 1)
        assert _host_chunk(n * W, sm) == LONG_CHUNK
        vals = rng.integers(1, B + 1, n, dtype=np.uint64)
        for nonzero in (LONG_CHUNK_MIN_ENTRIES - 1, LONG_CHUNK_MIN_ENTRIES):
            v = vals.copy()
            v[n // 2: n // 2 + n - nonzero] = 0
            col = _small_values(be, orc, v)
            _check(failures, orc, "plain 2^23, %d entries" % nonzero, srs24.params.commit(col), orc.commit_known_tau(col), be, nonzero + 2 * W * B)
        for k, tables in ((18, False), (19, True)):
            n = 1 << k
            c, W = be.msm_geometry(n, tables)
            B, BW = 1 << (c - 1), 1 if tables else W
            assert 24 <= _host_chunk(n * W, sm) <= 48
            v = rng.integers(1, B + 1, n, dtype=np.uint64)
            v[::7] = 0
            col = _small_values(be, orc, v)
            if tables:
                handle = ParamsKZG.from_bases(be, srs24.g()[:n]).precompute()
                got = handle.multiexp(col)
                del handle
            else:
                got = srs24.params.commit(col)
            _check(failures, orc, "%s 2^%d" % ("tabled" if tables else "plain", k), got, orc.commit_known_tau(col), be, int(np.count_nonzero(v)) + 2 * BW * B)
        assert not failures, "\n".join(failures)

    def test_more_giant_chains_than_giant_blocks(self, be, orc, srs24):
        """A range-check column (plain 2^22, values uniform in [1, V]): more than 256 buckets each hold between 25 and 4096
        chunks of entries, so msm_giant_kernel's 256 blocks loop over the queue."""
        n, V = 1 << 22, 3000
        c, W = be.msm_geometry(n, False)
        B = 1 << (c - 1)
        assert V <= B and n < LONG_CHUNK_MIN_ENTRIES       # one digit per value; M = n: the device uses the short chunk
        v = np.random.default_rng(0x6e0e).integers(1, V + 1, n, dtype=np.uint64)
        per_bucket = np.bincount(v.astype(np.int64))[1:]
        giants = int(((per_bucket >= (STITCH_CAP + 2) * SHORT_CHUNK) & (per_bucket <= HUGE_CHAIN * SHORT_CHUNK)).sum())
        assert giants > GIANT_BLOCKS, giants
        col = _small_values(be, orc, v)
        failures = []
        _check(failures, orc, "range check 2^22, V = %d" % V, srs24.params.commit(col), orc.commit_known_tau(col), be, n + 2 * W * B)
        assert not failures, "\n".join(failures)

    def test_k24_precompute_keeps_the_plain_layout_and_batch(self, be, orc, cols, srs24):
        """precompute() on the K = 24 SRS builds no tables when W x 2^24 x 64 B x 2 bases exceed a quarter of the device (80 GB
        H100: 24 GiB against 20 GiB). The ones column proves the geometry that ran; then a batch of three 2^24 columns that
        reuse the lanes' workspaces."""
        from spectre_b200.halo2 import BASIS_G
        c, W, BW = _tabled_geometry(be, NMAX, 2)
        srs24.params.precompute()
        failures = []
        _check(failures, orc, "K = 24 ones after precompute", srs24.params.commit(cols["ones"]), cols.known("ones", NMAX), be, NMAX + 2 * BW * (1 << (c - 1)))
        names = ("uniform", "witness", "minus_one")
        for name, got in zip(names, srs24.params.commit_batch(BASIS_G, [cols[nm] for nm in names])):
            _check(failures, orc, "K = 24 batch %s" % name, got, cols.known(name, NMAX))
        assert not failures, "\n".join(failures)


class TestOnTheK23SrsWithTables:
    """The aggregation circuit's SRS: K = 23 with window tables of both bases (one bucket set of c = 22 on an 80 GB H100)."""

    def test_chunk_threshold_with_tables(self, be, orc, srs23):
        """2^23 - 1 small values take the short-chunk fallback, 2^23 the long chunk: M pinned on both sides."""
        n = 1 << K23
        c, W, BW = _tabled_geometry(be, n, 2)
        B = 1 << (c - 1)
        vals = np.random.default_rng(0x6e10).integers(1, B + 1, n, dtype=np.uint64)
        failures = []
        for nonzero in (LONG_CHUNK_MIN_ENTRIES - 1, LONG_CHUNK_MIN_ENTRIES):
            v = vals.copy()
            v[: n - nonzero] = 0
            col = _small_values(be, orc, v)
            _check(failures, orc, "K = 23 tabled, %d entries" % nonzero, srs23.params.commit(col), orc.commit_known_tau(col), be, nonzero + 2 * BW * B)
        assert not failures, "\n".join(failures)

    def test_huge_chains_share_the_grid(self, be, orc, srs23):
        """all-(r - 1): with tables every window's digit lands in one bucket set, so each distinct digit magnitude is a huge
        chain and several share msm_huge_kernel's grid. A column whose every window holds the digit +B: one chain of about W x n
        entries in the last bucket."""
        n = 1 << K23
        c, W, BW = _tabled_geometry(be, n, 2)
        B = 1 << (c - 1)
        same, windows = _same_digit_scalar(c, W)
        assert _signed_digits(same, c, W) == windows
        failures = []
        for what, s, M in (("all-(r - 1)", R - 1, n * _signed_digits(R - 1, c, W)), ("every window +B", same, n * windows)):
            col = np.repeat(orc.fr([s]), n, axis=0)
            _check(failures, orc, "K = 23 tabled %s" % what, srs23.params.commit(col), orc.commit_known_tau(col), be, M + 2 * BW * B)
        assert not failures, "\n".join(failures)

    def test_batch_reuses_lanes_across_occupancies(self, be, orc, cols, srs23):
        """commit_batch_dev of seven 2^23 columns in the order uniform, zeros, ones, range check, all-(r - 1), witness-like,
        uniform: every lane runs consecutive MSMs with different bucket occupancy and chunk length over a bucket array that is
        never cleared. Each result against the known secret."""
        import torch
        from spectre_b200.halo2 import BASIS_G
        n = 1 << K23
        rng = np.random.default_rng(0x6e11)
        host = [cols["uniform"][:n], np.zeros((n, 4), dtype=np.uint64), cols["ones"][:n],
                _small_values(be, orc, rng.integers(1, 3001, n, dtype=np.uint64)), cols["minus_one"][:n], cols["witness"][:n],
                cols["uniform"][NMAX - n:]]
        dev = [torch.from_numpy(np.ascontiguousarray(h).view(np.int64)).cuda() for h in host]
        torch.cuda.synchronize()
        out = srs23.params.commit_batch_dev(BASIS_G, [d.data_ptr() for d in dev], n)
        del dev
        labels = ("uniform", "zeros", "ones", "range check", "all-(r - 1)", "witness-like", "second uniform")
        failures = []
        for label, h, got in zip(labels, host, out):
            _check(failures, orc, "K = 23 batch %s" % label, got, orc.commit_known_tau(h))
        assert not failures, "\n".join(failures)

    def test_commit_lagrange(self, be, orc, cols, srs23):
        a = cols["uniform"][: 1 << K23]
        assert np.array_equal(orc.g1_to_affine(srs23.params.commit_lagrange(a)), orc.commit_lagrange_known_tau(K23, a))
