"""CPU-only: the C-ABI library builds for sm_90a, loads, exports every symbol include/spectre_b200.h declares,
and refuses to run without a GPU (no CPU fallback). No compute calls here."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libpath():
    from spectre_b200 import build
    return build.build()


def declared_symbols():
    with open(os.path.join(ROOT, "include", "spectre_b200.h")) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(spb_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(libpath):
    syms = declared_symbols()
    assert len(syms) >= 40
    lib = ctypes.CDLL(libpath)
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, "declared in include/spectre_b200.h but not exported: %s" % missing


def test_rust_shim_binds_only_declared_and_exported_symbols(libpath):
    """shim/halo2_proofs_b200/src/b200.rs (the Rust `extern "C"` block a maintainer compiles on a cargo host) names only entry
    points the header declares and the library exports, with the argument count of the C declaration."""
    with open(os.path.join(ROOT, "shim", "halo2_proofs_b200", "src", "b200.rs")) as f:
        rust = f.read()
    block = rust[rust.index('extern "C" {'):]
    block = block[:block.index("\n}\n")]
    rust_fns = {m.group(1): m.group(2) for m in re.finditer(r"pub fn (spb_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->[^;]*)?;", block, flags=re.S)}
    assert len(rust_fns) >= 45
    with open(os.path.join(ROOT, "include", "spectre_b200.h")) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    lib = ctypes.CDLL(libpath)
    for name, args in rust_fns.items():
        assert hasattr(lib, name), "%s is bound by the Rust shim but not exported" % name
        m = re.search(r"\b%s\s*\((.*?)\)\s*;" % name, header, flags=re.S)
        assert m, "%s is bound by the Rust shim but not declared in the header" % name
        c_args = [a for a in m.group(1).split(",") if a.strip() and a.strip() != "void"]
        r_args = [a for a in args.split(",") if a.strip()]
        assert len(c_args) == len(r_args), "%s: %d C parameters, %d in the Rust declaration" % (name, len(c_args), len(r_args))


def test_only_abi_symbols_are_exported(libpath):
    out = subprocess.check_output(["nm", "-D", "--defined-only", libpath], text=True)
    exported = [l.split()[-1] for l in out.splitlines() if " T " in l]
    assert exported and all(s.startswith("spb_") for s in exported), exported


def test_cubin_is_sm_90a(libpath):
    out = subprocess.run(["cuobjdump", "-lelf", libpath], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_cpu_fallback_without_gpu(libpath):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here")
    from spectre_b200 import halo2
    with pytest.raises(halo2.BackendError):
        halo2.Backend([0])


def test_product_never_imports_oracle():
    """The product package must not reference the oracle (test infrastructure)."""
    pkg = os.path.join(ROOT, "spectre_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".hpp")):
                with open(os.path.join(dirpath, fn)) as f:
                    text = f.read()
                assert "halo2_oracle" not in text and "from oracle" not in text and "import oracle" not in text, fn
                assert "abi_shim" not in text and "spb_shim" not in text, fn      # the test-only CPU stand-in of the ABI


def test_product_library_has_no_cpu_stand_in(libpath):
    """libspectre_b200.so neither links nor embeds the oracle or the test-only ABI shim"""
    needed = subprocess.check_output(["readelf", "-d", libpath], text=True)
    assert "halo2_oracle" not in needed and "spb_shim" not in needed
    syms = subprocess.check_output(["nm", "-D", libpath], text=True)
    assert " orc_" not in syms


def _build_cpp_mirror(libpath, out_dir):
    """the executable goes to out_dir: the checkout may be read-only"""
    exe = os.path.join(str(out_dir), "host_mirror")
    src = os.path.join(ROOT, "tests", "cpp", "host_mirror.cpp")
    libdir = os.path.dirname(libpath)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, src, "-L" + libdir, "-lspectre_b200", "-Wl,-rpath," + libdir])
    return exe


def test_cpp_host_mirror_compiles_and_links(libpath, tmp_path):
    """include/spectre_b200.hpp (the compiled-language host side) builds against the C ABI."""
    exe = _build_cpp_mirror(libpath, tmp_path)
    assert subprocess.check_output([exe], text=True).strip() == "linked"


@pytest.mark.gpu
def test_cpp_host_mirror_runs(libpath, tmp_path):
    exe = _build_cpp_mirror(libpath, tmp_path)
    out = subprocess.run([exe, "run"], capture_output=True, text=True)
    assert out.returncode == 0 and "host mirror ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_error_paths_and_threads(libpath):
    """Errors come back as status codes with text; two Python threads can share one context."""
    import threading
    import numpy as np
    from spectre_b200 import halo2
    from oracle import oracle as orc
    orc.build(); orc.lib()
    be = halo2.Backend([0])
    k = 8
    params = halo2.ParamsKZG.setup(be, k, orc.srs_tau())
    too_long = orc.fr_random_chacha((1 << k) + 1, 1)
    with pytest.raises(AssertionError):
        params.commit(too_long)
    out = np.empty(12, dtype=np.uint64)
    rc = be.lib.spb_msm(be.ctx, params.h, 0, too_long.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(too_long.shape[0]), out.ctypes.data_as(ctypes.c_void_p))
    assert rc != 0 and b"SRS has" in be.lib.spb_last_error(be.ctx)
    rc = be.lib.spb_ntt(be.ctx, too_long.ctypes.data_as(ctypes.c_void_p), 29, too_long.ctypes.data_as(ctypes.c_void_p))
    assert rc != 0
    empty = params.commit(np.zeros((0, 4), dtype=np.uint64))
    assert not empty[8:].any()
    polys = [orc.fr_random_chacha(1 << k, 10 + i) for i in range(6)]
    want = [orc.commit_known_tau(p) for p in polys]
    results = [None] * len(polys)

    def work(i):
        results[i] = orc.g1_to_affine(params.commit(polys[i]))
    ts = [threading.Thread(target=work, args=(i,)) for i in range(len(polys))]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert all(np.array_equal(r, w) for r, w in zip(results, want))
    be.close()


def test_every_entry_point_survives_null_arguments(libpath):
    """`include/spectre_b200.h`: "nothing aborts or throws". Without a GPU no context exists, but every exported function must
    still refuse an all-NULL call (null context, null pointers, zero sizes) with an error code or a no-op instead of
    dereferencing -- each one is called in its own process so a crash is caught (spb_init is skipped: it would probe devices)."""
    import subprocess
    import sys
    out = subprocess.run(["nm", "-D", "--defined-only", libpath], capture_output=True, text=True, check=True).stdout
    names = sorted(l.split()[-1] for l in out.splitlines() if " T spb_" in l)
    assert len(names) > 80
    prog = ("import ctypes,sys; lib=ctypes.CDLL(%r)\n"
            "for n in sys.argv[1:]:\n"
            "    f=getattr(lib,n); f.restype=ctypes.c_int64; f(*([ctypes.c_void_p(0)]*16)); print('ok',n,flush=True)\n" % libpath)
    todo = [n for n in names if n != "spb_init"]
    p = subprocess.run([sys.executable, "-c", prog] + todo, capture_output=True, text=True, timeout=120)
    done = [l.split()[1] for l in p.stdout.splitlines() if l.startswith("ok ")]
    assert p.returncode == 0 and done == todo, "crashed in %s" % (todo[len(done)] if len(done) < len(todo) else p.stderr[-300:])
