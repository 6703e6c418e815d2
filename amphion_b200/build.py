"""Build libamphion_b200.so in-tree with nvcc for sm_90a (H100; no torch headers, plain C ABI).

Each .cu is compiled to an object in `_build/` (in parallel, only when it or a header changed) and the
objects are linked into the shared library next to this file, so the `.so` travels with the tree."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libamphion_b200.so")
SOURCES = ["ab_capi.cu", "ab_kernels_fp32.cu", "ab_kernels_tc.cu", "ab_mel.cu", "ab_pcm.cu", "ab_diffwave.cu", "ab_facodec.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC)")


def _headers() -> list[str]:
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(HERE), "include", "amphion_b200.h"))
    return hs


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + _headers()
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    hdr_t = max(os.path.getmtime(h) for h in _headers())
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]

    def compile_one(s: str) -> tuple[str, str]:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s[:-3] + ".o")
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(src)
                and os.path.getmtime(obj) > hdr_t):
            return obj, ""
        cmd = [nvcc, "-std=c++17", "-O3", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC", "-c", "-o", obj, src]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n" + r.stdout + r.stderr)
        return obj, r.stdout + r.stderr

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(compile_one, srcs))
    if verbose:
        for _, log in results:
            if log:
                print(log)
    # cuFFT by soname only: at run time the loader resolves libcufft.so.11 to the
    # copy torch already mapped (the same FFT backend torch.stft uses).
    cmd = [nvcc, "-shared", *ARCH, "-o", LIB] + [o for o, _ in results] + ["-L/usr/local/cuda/lib64", "-lcufft", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
