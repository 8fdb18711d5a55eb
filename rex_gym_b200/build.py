"""In-tree build of librexsim.so (hand-written sm_90a CUDA + the C ABI).  nvcc cross-compiles
without a GPU; the built .so is git-ignored but travels to the GPU box with the snapshot.

rexsim_kernel.cu is compiled once per (task, signal) pair (-DREXSIM_UNIT=k: only that pair's step kernels)
plus one unit for the reset / settle / state kernels; the units run in parallel and are linked into one .so."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "librexsim.so")
STAMP = os.path.join(HERE, "librexsim.srchash")
KERNEL_UNITS = [0, 1, 2, 3, 4, 5, 6, 7, 100]           # see the tail of rexsim_kernel.cu
OTHER_SOURCES = ["rexsim_capi.cu", "rexsim_agent.cu", "rexsim_render.cu"]
HEADERS = ["rexsim_kernel.cuh", "rexsim_arm.cuh", "rexsim_host.h", os.path.join("..", "..", "include", "rexsim.h"),
           os.path.join("..", "..", "include", "rexsim_agent.h"), os.path.join("..", "..", "include", "rexsim_recurrent.h")]
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17"]
NVCC_FLAGS = ARCH_FLAGS + ["-Xcompiler", "-fPIC"]


def _source_hash():
    h = hashlib.sha256()
    for f in ["rexsim_kernel.cu"] + OTHER_SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(repr(KERNEL_UNITS).encode())
    return h.hexdigest()


def needs_build():
    """Content-based (not mtime-based: snapshots copied to the GPU box do not have to preserve mtimes)."""
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    return open(STAMP).read().strip() != _source_hash()


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.returncode, r.stdout, cmd


def build(force=False, verbose=False, variant=None, defines=(), units=None):
    """variant / defines: developer A/B builds -- librexsim_<variant>.so compiled with extra -D flags, loaded through
    REXSIM_LIB (rex_gym_b200/_capi.py); the product library is the plain call."""
    if variant:
        return _build_variant(variant, list(defines), verbose, units)
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ, exist_ok=True)
    extra = ["-Xptxas", "-v"] if verbose else []
    jobs, objs = [], []
    for u in KERNEL_UNITS:
        o = os.path.join(OBJ, "kernel_u%d.o" % u)
        objs.append(o)
        jobs.append([nvcc] + NVCC_FLAGS + extra + ["-DREXSIM_UNIT=%d" % u, "-c", os.path.join(CSRC, "rexsim_kernel.cu"), "-o", o])
    for f in OTHER_SOURCES:
        o = os.path.join(OBJ, f.replace(".cu", ".o"))
        objs.append(o)
        jobs.append([nvcc] + NVCC_FLAGS + extra + ["-c", os.path.join(CSRC, f), "-o", o])
    workers = int(os.environ.get("REXSIM_BUILD_JOBS", "0")) or min(len(jobs), os.cpu_count() or 4)
    with ThreadPoolExecutor(workers) as ex:
        results = list(ex.map(_run, jobs))
    out = ""
    for rc, log, cmd in results:
        out += log
        if rc != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + log)
            raise RuntimeError("nvcc failed building librexsim.so")
    rc, log, cmd = _run([nvcc] + ARCH_FLAGS + ["-shared", "-o", LIB] + objs)
    if rc != 0:
        sys.stderr.write(log)
        raise RuntimeError("link of librexsim.so failed")
    if verbose:
        print(out)
    with open(STAMP, "w") as f:
        f.write(_source_hash())
    return LIB


def _build_variant(variant, defines, verbose, units=None):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    obj = os.path.join(OBJ, variant)
    os.makedirs(obj, exist_ok=True)
    lib = os.path.join(HERE, "librexsim_%s.so" % variant)
    extra = (["-Xptxas", "-v"] if verbose else []) + ["-D" + d for d in defines]
    jobs, objs = [], []
    for u in KERNEL_UNITS:
        o = os.path.join(obj, "kernel_u%d.o" % u)
        objs.append(o)
        if units is not None and u not in units and os.path.exists(os.path.join(OBJ, "kernel_u%d.o" % u)):
            objs[-1] = os.path.join(OBJ, "kernel_u%d.o" % u)       # untouched units: reuse the product objects
            continue
        jobs.append([nvcc] + NVCC_FLAGS + extra + ["-DREXSIM_UNIT=%d" % u, "-c", os.path.join(CSRC, "rexsim_kernel.cu"), "-o", o])
    for f in OTHER_SOURCES:
        objs.append(os.path.join(OBJ, f.replace(".cu", ".o")))
    with ThreadPoolExecutor(min(len(jobs), os.cpu_count() or 4)) as ex:
        results = list(ex.map(_run, jobs))
    for rc, log, cmd in results:
        if verbose:
            print(log)
        if rc != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + log)
            raise RuntimeError("nvcc failed building " + lib)
    rc, log, cmd = _run([nvcc] + ARCH_FLAGS + ["-shared", "-o", lib] + objs)
    if rc != 0:
        sys.stderr.write(log)
        raise RuntimeError("link failed: " + lib)
    return lib


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("-v", action="store_true")
    ap.add_argument("--variant")
    ap.add_argument("-D", action="append", default=[])
    ap.add_argument("--units", type=lambda t: [int(x) for x in t.split(",")])
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.v, variant=a.variant, defines=a.D, units=a.units))
