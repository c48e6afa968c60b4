"""In-tree build of the sm_90a kernel library (nvcc -> occdepth_b200/lib/libocc_b200.so).

No torch extension machinery: the product boundary is a plain C ABI (include/occdepth_b200.h), so the
library is compiled with nvcc directly and loaded through ctypes (occdepth_b200/_lib.py).
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIBNAME = "libocc_b200.so"
HEADERS = ("occdepth_b200.h", "occdepth_b200_comm.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build occdepth_b200 kernels")
    return nvcc


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        h.update(f.read())
    for hdr in sorted(os.listdir(CSRC)):
        if hdr.endswith((".cuh", ".h")):
            with open(os.path.join(CSRC, hdr), "rb") as f:
                h.update(f.read())
    for hdr in HEADERS:
        with open(os.path.join(HERE, "..", "include", hdr), "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def lib_path():
    return os.path.join(LIBDIR, LIBNAME)


def build(verbose=False, force=False):
    """Compile every csrc/*.cu for sm_90a and link lib/libocc_b200.so (incremental by content hash)."""
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()
    srcs = _sources()
    jobs = []
    objs = []
    for src in srcs:
        base = os.path.splitext(os.path.basename(src))[0]
        obj = os.path.join(OBJDIR, base + ".o")
        stamp = obj + ".sha1"
        dig = _digest(src)
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.exists(stamp)
                and open(stamp).read().strip() == dig):
            continue
        jobs.append((src, obj, stamp, dig))

    def compile_one(job):
        src, obj, stamp, dig = job
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = obj + ".log"
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout + r.stderr))
        with open(stamp, "w") as f:
            f.write(dig)
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    out = lib_path()
    if jobs or not os.path.exists(out):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out] + objs + ["-ldl"]   # NCCL is loaded at run time (csrc/comm.cu)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    build_occd_run(nvcc, force=jobs or force)
    return out


def occd_run_path():
    return os.path.join(LIBDIR, "occd_run")


def build_occd_run(nvcc, force=False):
    """tools/occd_run.c: a plain C program linked against libocc_b200.so (found next to it) and the CUDA runtime"""
    src = os.path.join(HERE, "..", "tools", "occd_run.c")
    hdr = os.path.join(HERE, "..", "include", "occdepth_b200.h")
    h = hashlib.sha1()
    for p in [src] + [os.path.join(HERE, "..", "include", x) for x in HEADERS]:
        with open(p, "rb") as f:
            h.update(f.read())
    exe, stamp = occd_run_path(), occd_run_path() + ".sha1"
    if not force and os.path.exists(exe) and os.path.exists(stamp) and open(stamp).read().strip() == h.hexdigest():
        return exe
    cmd = [nvcc, "-O2", "-x", "c", src, "-I", os.path.dirname(hdr), "-L", LIBDIR, "-locc_b200",
           "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("occd_run build failed:\n" + r.stdout + r.stderr)
    with open(stamp, "w") as f:
        f.write(h.hexdigest())
    return exe


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
