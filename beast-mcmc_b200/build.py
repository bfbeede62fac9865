"""In-tree build of the engine's shared libraries with nvcc for sm_90a (H100).

  beast-mcmc_b200/csrc/libhmsbeagle.so      the C ABI (include/libhmsbeagle_b200.h), CUDA runtime linked statically
  beast-mcmc_b200/csrc/libhmsbeagle-jni.so  the JNI shim BEAST's lib/beagle.jar binds (System.loadLibrary("hmsbeagle-jni"))
  oracle/liboracle_cpu.so                   the CPU restatement used as checker / cpu_baseline (test infrastructure)

The .so files are git-ignored build products.  So that a binary left in the tree can never silently drift from the
sources, a SHA-256 over the engine's sources is compiled into the library (``b200GetSourceHash``,
also the build-metadata suffix of ``beagleGetVersion``) and written next to it; ``build_engine`` rebuilds whenever the
recorded hash differs from the sources' and ``verify_engine`` asserts the LOADED library reports the current hash.
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
ENGINE_UNITS = ("api.cu", "kernels.cu", "walk4e.cu", "incr.cu", "multi.cu", "patterns.cu", "ancestral.cu")
ENGINE_HEADERS = (os.path.join(CSRC, "engine.h"), os.path.join(CSRC, "walk4.cuh"), os.path.join(CSRC, "multi.h"),
                  os.path.join(ROOT, "include", "libhmsbeagle_b200.h"))


def _engine_units():
    return [os.path.join(CSRC, f) for f in ENGINE_UNITS if os.path.exists(os.path.join(CSRC, f))]


def source_hash() -> str:
    h = hashlib.sha256()
    for path in sorted(_engine_units()) + sorted(ENGINE_HEADERS):
        h.update(os.path.basename(path).encode() + b"\0")
        h.update(open(path, "rb").read())
    return h.hexdigest()[:16]


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("build failed: " + " ".join(cmd))
    if verbose and (r.stdout or r.stderr):
        print(r.stdout + r.stderr)


def lib_path(name="libhmsbeagle.so"):
    return os.path.join(CSRC, name)


def build_engine(force=False, verbose=False):
    out = lib_path()
    stamp = out + ".srchash"
    want = source_hash()
    have = open(stamp).read().strip() if os.path.exists(stamp) and os.path.exists(out) else None
    if not force and have == want:
        return out
    if not os.path.exists(NVCC):
        raise RuntimeError(f"{out} is stale (sources {want}, binary {have}) and nvcc is not available to rebuild it")
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    common = [NVCC, *ARCH, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden",
              "-Xptxas", "-v" if verbose else "-O3"]

    def compile_unit(src):
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        extra = [f'-DB200_SOURCE_HASH="{want}"'] if src.endswith("api.cu") else []
        # api.cu carries the hash of ALL sources: it is recompiled whenever anything changed
        if force or extra or _stale(obj, [src, *ENGINE_HEADERS]):
            _run([*common, *extra, "-c", "-o", obj, src], verbose)
        return obj

    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_unit, _engine_units()))
    _run([NVCC, *ARCH, "-shared", "-cudart", "static", "-Xcompiler", "-fPIC", "-o", out, *objs, "-lpthread"], verbose)
    with open(stamp, "w") as f:
        f.write(want + "\n")
    return out


def verify_engine():
    """The library that actually loads must have been built from the sources in this tree."""
    import ctypes
    lib = ctypes.CDLL(lib_path())
    lib.b200GetSourceHash.restype = ctypes.c_char_p
    got, want = lib.b200GetSourceHash().decode(), source_hash()
    if got != want:
        raise RuntimeError(f"libhmsbeagle.so was built from other sources (binary {got}, tree {want}): rebuild")
    return got


def build_jni(force=False, verbose=False):
    src = os.path.join(CSRC, "jni_shim.cpp")
    if not os.path.exists(src):
        return None
    out = lib_path("libhmsbeagle-jni.so")
    deps = [src, os.path.join(ROOT, "include", "jni_min.h"), os.path.join(ROOT, "include", "libhmsbeagle_b200.h")]
    if force or _stale(out, deps):
        _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-I", os.path.join(ROOT, "include"),
              "-o", out, src, "-L", CSRC, "-lhmsbeagle", "-Wl,-rpath,$ORIGIN"], verbose)
    return out


def build_oracle(force=False, verbose=False):
    src = os.path.join(ROOT, "oracle", "beagle_cpu.c")
    if not os.path.exists(src):
        return None
    out = os.path.join(ROOT, "oracle", "liboracle_cpu.so")
    if force or _stale(out, [src]):
        # no -march=native: the binary travels to a different host CPU; the hot loops carry target_clones instead
        _run(["gcc", "-O3", "-std=gnu11", "-fPIC", "-shared", "-pthread", "-o", out, src, "-lm"], verbose)
    return out


def build_cdriver(force=False, verbose=False):
    """bench infrastructure (harness/cdriver.c): replays prepared C-ABI call sequences from C, as a JVM's JNI thread would."""
    src = os.path.join(ROOT, "harness", "cdriver.c")
    if not os.path.exists(src):
        return None
    out = os.path.join(ROOT, "harness", "libcdriver.so")
    if force or _stale(out, [src, os.path.join(ROOT, "include", "libhmsbeagle_b200.h"), lib_path()]):
        _run(["gcc", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-o", out, src, "-L", CSRC, "-lhmsbeagle",
              "-Wl,-rpath,$ORIGIN/../beast-mcmc_b200/csrc"], verbose)
    return out


def build_all(force=False, verbose=False):
    return (build_engine(force, verbose), build_jni(force, verbose), build_oracle(force, verbose),
            build_cdriver(force, verbose))


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print("source hash", verify_engine())
