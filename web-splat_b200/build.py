"""Builds libwebsplat_b200.so (sm_90a only, i.e. H100) in-tree with nvcc.

Every translation unit is compiled with
    -gencode arch=compute_90a,code=sm_90a -lineinfo -O3
preprocess.cu additionally with -fmad=false (stage 1 is bit-exact against the CPU oracle:
one IEEE rounding per written operation; the kernel is HBM-bound, so this costs nothing).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libwebsplat_b200.so")
OBJ = os.path.join(HERE, "build")

COMMON = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-Xptxas", "-v", "-Xptxas", "-warn-spills",
]
UNITS = {
    "preprocess.cu": ["-fmad=false"],
    "radix_sort.cu": [],
    "binning.cu": [],
    "composite.cu": [],
    "shard.cu": [],
    "ingest.cu": ["-fmad=false"],
    "capi.cu": [],
}
HEADERS = ["ws_device.cuh", "ws_kernels.h", os.path.join("..", "..", "include", "websplat_b200.h")]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    jobs = []
    objs = []
    for src, extra in UNITS.items():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            jobs.append((src, [_nvcc()] + COMMON + extra + ["-c", s, "-o", o]))

    def run(job):
        name, cmd = job
        p = subprocess.run(cmd, capture_output=True, text=True)
        return name, p.returncode, p.stdout + p.stderr

    logs = {}
    with ThreadPoolExecutor(max_workers=len(UNITS)) as ex:
        for name, rc, log in ex.map(run, jobs):
            logs[name] = log
            if rc != 0:
                sys.stderr.write(log)
                raise RuntimeError("nvcc failed on %s" % name)
            if verbose:
                sys.stderr.write(log)
    if jobs or force or _stale(OUT, objs):
        cmd = [_nvcc(), "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError("link failed")
    try:                                   # the C++ tool is auxiliary: the library must not depend on it
        build_tools(force=force)
    except Exception as e:                 # noqa: BLE001
        sys.stderr.write("websplat_b200: tools/ws_render.cpp was not built: %s\n" % e)
    return OUT, logs


TOOLS_DIR = os.path.normpath(os.path.join(HERE, "..", "tools"))
TOOL_OUT = os.path.join(HERE, "ws_render")


def build_tools(force=False):
    """tools/ws_render.cpp: the offline dataset renderer in C++ on top of the C ABI (header-only mirror include/websplat_b200.hpp)."""
    src = os.path.join(TOOLS_DIR, "ws_render.cpp")
    inc = os.path.normpath(os.path.join(HERE, "..", "include"))
    deps = [src, os.path.join(TOOLS_DIR, "npz_reader.hpp"), os.path.join(inc, "websplat_b200.hpp"), os.path.join(inc, "websplat_b200.h"), OUT]
    if not os.path.exists(src):
        return None
    if force or _stale(TOOL_OUT, deps):
        cxx = os.environ.get("CXX") or ("/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++")
        have_zlib = any(os.path.exists(os.path.join(d, "zlib.h")) for d in ("/usr/include", "/usr/local/include"))
        cmd = [cxx, "-std=c++17", "-O2", "-Wall", "-Wextra", "-o", TOOL_OUT, src, "-L" + HERE, "-lwebsplat_b200",
               "-Wl,-rpath,$ORIGIN", "-ldl", "-lpthread", "-lrt"]
        if have_zlib:                      # deflated .npz members (np.savez_compressed); stored ones need nothing
            cmd += ["-DWS_HAVE_ZLIB", "-lz"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError("building tools/ws_render.cpp failed")
        if p.stderr.strip():
            sys.stderr.write(p.stderr)
    return TOOL_OUT


if __name__ == "__main__":
    out, logs = build(force="--force" in sys.argv, verbose=True)
    print(out)
