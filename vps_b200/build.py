"""Build libvps_b200.so (the C-ABI kernel library) in-tree with nvcc for sm_90a (H100).

Incremental: each csrc/*.cu is compiled to build/*.o only when it (or a header) is newer than the
object; objects are linked into vps_b200/lib/libvps_b200.so.  No GPU is needed (cross-compile).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
OBJ = os.path.join(ROOT, "build")
LIBDIR = os.path.join(ROOT, "lib")
LIB = os.path.join(LIBDIR, "libvps_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _newer(src_list, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(ROOT, "..", "include", "vps_b200.h"))
    nvcc = _nvcc()
    jobs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s[:-3] + ".o")
        if force or _newer([src] + hdrs, obj):
            jobs.append((src, obj))

    def run(job):
        src, obj = job
        cmd = [nvcc] + NVCC_FLAGS + os.environ.get("VPS_NVCC_EXTRA", "").split() + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return job, r

    failed = False
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for (src, obj), r in ex.map(run, jobs):
            log = os.path.join(OBJ, os.path.basename(src) + ".log")
            with open(log, "w") as f:
                f.write(r.stdout + r.stderr)
            if r.returncode != 0:
                failed = True
                sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, r.stderr[-6000:]))
            elif verbose:
                sys.stderr.write(r.stderr)
    if failed:
        raise RuntimeError("vps_b200: CUDA build failed")
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in srcs]
    if force or jobs or _newer(objs, LIB):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                      "-lcudart_static", "-Xlinker", "--no-undefined", "-lpthread",
                                                      "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("vps_b200: link failed:\n" + r.stderr[-4000:])
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
