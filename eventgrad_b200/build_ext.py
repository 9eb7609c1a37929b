"""Build the sm_90a (H100) extension in-tree: eventgrad_b200/_C*.so.

nvcc cross-compiles without a GPU; the built .so is git-ignored and rebuilt from csrc/ on demand.
No torch headers are involved, so a full rebuild takes a few seconds; objects are cached by source
mtime under csrc/build/.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(CSRC, "build")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH_FLAGS + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                           "--expt-relaxed-constexpr", "-Xptxas", "-v"]
CU_SOURCES = ["gossip.cu", "gossip_dbuf.cu", "gossip_graph.cu", "gossip_q8.cu", "gossip_gt.cu", "gossip_ed.cu", "gossip_rounds.cu", "gossip_match.cu", "ce_push.cu", "allreduce.cu", "allreduce_nvls.cu", "sparse.cu", "augment.cu", "ipc.cu", "bn_act.cu", "bn_nchw.cu", "linear_tc_tma.cu", "conv_tc.cu"]
CPP_SOURCES = ["bindings.cpp"]
HEADERS = ["api.h", "common.cuh", "bn_common.cuh", "host_loader.h", "tc_common.cuh"]


def so_path() -> str:
    ext = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return os.path.join(HERE, "_C" + ext)


def _cudart_dirs():
    dirs = []
    try:
        import nvidia.cuda_runtime  # torch's bundled runtime wheel
        dirs.append(os.path.join(os.path.dirname(nvidia.cuda_runtime.__file__), "lib"))
    except Exception:
        pass
    dirs.append(os.path.join(CUDA_HOME, "lib64"))
    return [d for d in dirs if os.path.isdir(d)]


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd, log):
    r = subprocess.run(cmd, capture_output=True, text=True)
    log.append("$ " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("build failed:\n" + log[-1])


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile what is stale and link the extension.  Safe under torchrun: ranks serialise on a file lock (the first
    one builds, the others find everything fresh) and the .so is linked to a temp name and renamed into place."""
    import fcntl
    os.makedirs(BUILD, exist_ok=True)
    with open(os.path.join(BUILD, ".lock"), "w") as lk:
        fcntl.flock(lk, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lk, fcntl.LOCK_UN)


def _build_locked(force: bool, verbose: bool) -> str:
    nvcc = os.path.join(CUDA_HOME, "bin", "nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc") or nvcc
    import pybind11
    py_inc = [sysconfig.get_paths()["include"], pybind11.get_include()]
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    log, jobs, objs = [], [], []
    for src in CU_SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(BUILD, src + ".o")
        objs.append(obj)
        twin = {"gossip_dbuf.cu": "gossip.cu", "gossip_graph.cu": "gossip.cu", "gossip_q8.cu": "gossip.cu",
                "gossip_gt.cu": "gossip.cu", "gossip_ed.cu": "gossip.cu", "gossip_match.cu": "gossip.cu",
                "allreduce_nvls.cu": "allreduce.cu"}.get(src)   # second compile of the same source
        deps = [sp] + hdrs + ([os.path.join(CSRC, twin)] if twin else [])
        if force or _stale(obj, deps):
            jobs.append([nvcc] + NVCC_FLAGS + ["-I", CSRC, "-c", sp, "-o", obj])
    for src in CPP_SOURCES:
        sp = os.path.join(CSRC, src)
        obj = os.path.join(BUILD, src + ".o")
        objs.append(obj)
        if force or _stale(obj, [sp] + hdrs):
            jobs.append(["g++", "-O2", "-fPIC", "-std=c++17", "-fvisibility=hidden",
                         "-I", CSRC, "-I", os.path.join(CUDA_HOME, "include")]
                        + sum([["-I", i] for i in py_inc], []) + ["-c", sp, "-o", obj])
    with ThreadPoolExecutor(max_workers=8) as ex:
        list(ex.map(lambda c: _run(c, log), jobs))
    out = so_path()
    if jobs or force or not os.path.exists(out):
        rdirs = _cudart_dirs()
        tmp = out + f".tmp{os.getpid()}"
        link = ["g++", "-shared", "-o", tmp] + objs
        for d in rdirs:
            link += ["-L", d, f"-Wl,-rpath,{d}"]
        link += ["-l:libcudart.so.12", "-lpthread"]
        _run(link, log)
        os.replace(tmp, out)
    with open(os.path.join(BUILD, "build.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return out


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built", p)
