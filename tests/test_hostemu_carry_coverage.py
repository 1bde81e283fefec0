"""CPU-only: the operand corpus of tests/arith_corpus.py drives every carry of the device field arithmetic
(spectre_b200/csrc/field.cuh), and every carry the code throws away is zero unless it is thrown away on purpose.

The corpus runs through the carry-trace build of the emulated PTX path (ptx.cuh under SPB_EMULATE_PTX_TRACE), one field
and one primitive at a time:
  * carry in: every instruction in field.cuh that reads CF (addc*, subc*, madc*) saw CF = 0 and CF = 1 over the
    primitives of a field, unless CONSTANT_CF below says why the flag cannot change there;
  * discarded carry out: every addc, subc and last madc_wide link discards a zero carry, except at the INTENTIONAL_WRAPS,
    which must also be seen wrapping -- this is what the bound comments in field.cuh claim ("no carry out", "never
    carries out", "carry-out proven zero by the caller"), checked on the corpus;
  * value: every result equals the Python integer one.
Sites are found by reading field.cuh, so a carry instruction added there without corpus coverage or an entry below fails
here with its file and line.
"""
import re

import numpy as np
import pytest

from tests import arith_corpus as ac

FIELDS = ("fr", "fq")

# (source text that identifies the line, reason) -- the line's discarded carry out is 1 on purpose for some inputs
INTENTIONAL_WRAPS = [
    ("uint32_t borrow = ptx::subc(0, 0);", "subc(0, 0) materialises the borrow of the chain above it as 0 or all-ones"),
    ("const uint32_t borrow = ptx::subc(0u, 0u);", "subc(0, 0) materialises the borrow of a*b - c*d as 0 or all-ones"),
    ("r.l[7] = ptx::addc(r.l[7], P::mod(7) & borrow);", "fp_sub adds m back after a borrow: a - b + m wraps past 2^256"),
    ("t[15] = ptx::addc(t[15], P::mod(7) & borrow);", "fp_mul_sub_mul's borrow correction adds m * 2^256 to a difference held mod 2^512"),
]
# (source text, reason) -- a CF-reading line whose flag is the same for every operand of every primitive. None in field.cuh:
# every carry chain there both carries and does not over the corpus.
CONSTANT_CF = []

CF_READERS = {"ptx::addc": "addc", "ptx::addc_cc": "addc_cc", "ptx::subc": "subc", "ptx::subc_cc": "subc_cc", "ptx::madc_wide": "madc_wide",
              "ptx::madc_wide_cc": "madc_wide_cc", "SPB_MADC_CC": "madc_wide_cc", "SPB_MADC_TOP": "madc_wide"}
DROPPERS = ("addc", "subc", "madc_wide")


def _source():
    with open(ac.FIELD_H) as f:
        return f.read().splitlines()


def device_sites():
    """{(line, instruction)} of every CF-reading call in the 32-bit-limb (device) part of field.cuh"""
    lines = _source()
    lo = next(i for i, l in enumerate(lines) if l.startswith("#if defined(SPB_LIMB32_PATH)"))
    hi = next(i for i, l in enumerate(lines) if l.startswith("// 64-bit limb path"))
    sites = set()
    for i in range(lo, hi):
        text = lines[i].strip()
        if text.startswith("#define") or text.startswith("//"):
            continue
        for m in re.finditer(r"(ptx::\w+|SPB_MADC_CC|SPB_MADC_TOP)\s*\(", text):
            if m.group(1) in CF_READERS:
                sites.add((i + 1, CF_READERS[m.group(1)]))
    return sites


def _lines_of(entries):
    """source text -> line numbers (every entry must still name a line of field.cuh)"""
    lines = _source()
    out = {}
    for text, reason in entries:
        hits = [i + 1 for i, l in enumerate(lines) if text in l]
        assert hits, "allowlist entry no longer matches a line of field.cuh: %r" % text
        for h in hits:
            out[h] = reason
    return out


def field_traces(lib, field, out_dir):
    """{primitive: per-line trace of the corpus} for one field"""
    return {prim: ac.by_line({k: v for k, v in ac.trace_of(lib, field, prim, ac.corpus(out_dir, field, prim)).items()
                              if k[0] == "field.cuh"})
            for prim in ac.PRIMITIVES}


def coverage_failures(traces):
    """the violations of the three carry rules in per-primitive, per-line traces of one field, as readable lines"""
    wraps, constant = _lines_of(INTENTIONAL_WRAPS), _lines_of(CONSTANT_CF)
    seen = {}
    for tr in traces.values():
        for (_, line, op), bits in tr.items():
            seen[(line, op)] = seen.get((line, op), 0) | bits
    bad = []
    for line, op in sorted(device_sites()):
        bits = seen.get((line, op), 0)
        if not bits:
            bad.append("field.cuh:%d %s: never executed by the corpus" % (line, op))
        elif (bits & 3) != 3 and line not in constant:
            bad.append("field.cuh:%d %s: carry in only ever %d" % (line, op, 1 if bits & ac.TRACE_CF_IN1 else 0))
        if op in DROPPERS and line in wraps and bits and not bits & ac.TRACE_DROP1:
            bad.append("field.cuh:%d %s: the intentional wrap (%s) is never reached" % (line, op, wraps[line]))
    for prim, tr in traces.items():
        for (_, line, op), bits in sorted(tr.items()):
            if (line, op) not in device_sites():
                bad.append("field.cuh:%d %s: a carry site the source scan does not know" % (line, op))
            if bits & ac.TRACE_DROP1 and line not in wraps:
                bad.append("field.cuh:%d %s: %s discards a carry out of 1" % (line, op, prim))
    return bad


@pytest.fixture(scope="module")
def trace_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("hostemu_trace")
    return d, ac.build_hostemu(d, "trace")


def test_source_scan_finds_the_carry_chains():
    """the scan sees the chains the rules are about (a scan that found nothing would pass every rule)"""
    sites = device_sites()
    ops = {op for _, op in sites}
    assert ops == {"addc", "addc_cc", "subc", "subc_cc", "madc_wide", "madc_wide_cc"}
    assert len(sites) >= 60
    assert set(_lines_of(INTENTIONAL_WRAPS)) <= {line for line, _ in sites}


@pytest.mark.parametrize("field", FIELDS)
def test_corpus_drives_every_carry(trace_lib, field, capsys):
    out_dir, lib = trace_lib
    traces = field_traces(lib, field, out_dir)
    constant = _lines_of(CONSTANT_CF)
    with capsys.disabled():
        for prim, tr in traces.items():
            both = sum(1 for (_, line, _), bits in tr.items() if bits & 3 == 3)
            allow = sum(1 for (_, line, _), bits in tr.items() if bits & 3 != 3 and line in constant)
            print("\n%s %-11s %3d operand tuples, %3d carry sites reached, %3d saw CF = 0 and 1, %d allowlisted"
                  % (field, prim, len(ac.corpus(out_dir, field, prim)), len(tr), both, allow), end="")
    bad = coverage_failures(traces)
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("field", FIELDS)
def test_corpus_values_match_python(trace_lib, field):
    """the emulated device algorithm and the 64-bit host path give the Python integer result on the whole corpus"""
    out_dir, lib = trace_lib
    native = ac.build_hostemu(out_dir, "native")
    for prim in ac.PRIMITIVES:
        tuples = ac.corpus(out_dir, field, prim)
        want = [ac.expected(field, prim, t) for t in tuples]
        for name, l in (("ptx trace build", lib), ("64-bit host build", native)):
            got = ac.ints(ac.run_host(l, field, prim, tuples))
            bad = [(t, g, w) for t, g, w in zip(tuples, got, want) if g != w]
            assert not bad, "%s %s %s: %d wrong, first %r" % (name, field, prim, len(bad), bad[0])


def test_trace_build_computes_what_the_plain_emulation_does(trace_lib):
    """the trace records and changes nothing: its limbs are the plain SPB_EMULATE_PTX build's on the corpus"""
    out_dir, lib = trace_lib
    plain = ac.build_hostemu(out_dir, "ptx")
    for field in FIELDS:
        for prim in ac.PRIMITIVES:
            tuples = ac.corpus(out_dir, field, prim)
            assert np.array_equal(ac.run_host(lib, field, prim, tuples), ac.run_host(plain, field, prim, tuples)), (field, prim)


def test_an_uncovered_site_is_named(trace_lib):
    """the failure report is actionable: with the corpus of a*b - c*d cut down to its special values, the lines it no longer
    drives are reported as field.cuh:<line>"""
    out_dir, lib = trace_lib
    fams = [f for f in ac.families("fq", "mul_sub_mul") if f[0] == "special"]
    cut = ac.select(lib, "fq", "mul_sub_mul", [(name, c[:1]) for name, c in fams])
    tr = ac.by_line({k: v for k, v in ac.trace_of(lib, "fq", "mul_sub_mul", cut).items() if k[0] == "field.cuh"})
    bad = coverage_failures({"mul_sub_mul": tr})
    assert bad and all(re.match(r"field\.cuh:\d+ \w+: ", b) for b in bad)
    assert any("never executed" in b for b in bad)      # fp_add / fp_sub / fp_neg lines: not reached by a*b - c*d at all
