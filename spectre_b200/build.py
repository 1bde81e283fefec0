"""Build libspectre_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m spectre_b200.build [--force] [--verbose]

The .so is a build product (git-ignored); build() of __graft_entry__ makes it.
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# A/B experiments: SPB_BUILD_VARIANT=name SPB_BUILD_FLAGS="-DX ..." builds libspectre_b200_name.so next to the product
# library (select it at run time with SPB_LIB_PATH); the product is always the plain name with no extra flags.
VARIANT = os.environ.get("SPB_BUILD_VARIANT", "")
EXTRA_FLAGS = os.environ.get("SPB_BUILD_FLAGS", "").split() if VARIANT else []
OUT = os.path.join(HERE, "libspectre_b200%s.so" % ("_" + VARIANT if VARIANT else ""))
OBJDIR = os.path.join(HERE, "_obj" + ("_" + VARIANT if VARIANT else ""))
SOURCES = ["capi.cu", "ntt.cu", "msm.cu", "poly.cu", "quotient.cu", "lookup.cu", "plonk.cu", "witness.cu", "pairing.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr", "-cudart", "static"]


def _deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "spectre_b200.h")]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(p) > t for p in _deps())


def _compile(src, verbose):
    obj = os.path.join(OBJDIR, src.replace(".cu", ".o"))
    cmd = [NVCC] + FLAGS + EXTRA_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, r.stderr


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    with concurrent.futures.ThreadPoolExecutor(max_workers=len(srcs)) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if verbose:
        for _, log in results:
            sys.stderr.write(log)
    objs = [o for o, _ in results]
    cmd = [NVCC, "-shared", "-cudart", "static", "-o", OUT] + objs + ["-Xcompiler", "-fvisibility=hidden"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
