"""In-tree build of the C-ABI library (csrc/libwlk_b200.so) with nvcc for sm_90a."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libwlk_b200.so")
SOURCES = ["engine.cu", "kernels.cu", "gemm_simt.cu", "gemm_tc.cu", "attn_tc.cu", "qwen.cu", "qwen_text.cu", "diar.cu", "vad.cu", "sortformer.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-Wno-subobject-linkage", "--expt-relaxed-constexpr"]
# ptxas reports per kernel; its C7510 note means every wgmma.mma_async of a kernel was serialized (each MMA waits for
# the previous one to retire) because a function call is reachable while a wgmma group is in flight
PTXAS_FLAGS = ["-Xptxas", "-v"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def serialized_wgmma(ptxas_log: str) -> list[str]:
    """The lines of a ptxas log that report serialized wgmma pipelines (C7510)."""
    return [ln.strip() for ln in ptxas_log.splitlines() if "C7510" in ln]


def _run(cmd, verbose: bool) -> str:
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    return r.stdout + r.stderr


def compile_object(src: str, obj: str, nvcc: str | None = None, extra_flags=(), verbose: bool = False) -> None:
    """nvcc -c src -o obj for sm_90a.  Fails (and leaves no object behind, so the next build retries) when ptxas
    serialized the wgmma pipeline of any kernel in it."""
    log = _run([nvcc or _nvcc(), *NVCC_FLAGS, *PTXAS_FLAGS, *extra_flags, "-c", src, "-o", obj], verbose)
    bad = serialized_wgmma(log)
    if bad:
        if os.path.exists(obj):
            os.remove(obj)
        raise RuntimeError(f"ptxas serialized the wgmma pipeline in {os.path.basename(src)} (a function call is "
                           "reachable while a wgmma group is in flight):\n" + "\n".join(bad))


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "wlk_b200.h"))
    objs, jobs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(CSRC, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append((s, o))

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(lambda j: compile_object(*j, nvcc=nvcc, verbose=verbose), jobs))
    if jobs or force or _stale(LIB, objs):
        _run([nvcc, "-shared", "-o", LIB, *objs], verbose)  # static cudart (nvcc default)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
