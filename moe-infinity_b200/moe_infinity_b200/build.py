"""Build libb2m.so (sm_90a only) in-tree with nvcc.  `python -m moe_infinity_b200.build`."""
from __future__ import annotations

import os
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(PKG_DIR), "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libb2m.so")
SOURCES = ["grouped_gemm.cu", "route.cu", "ep.cu", "f32_path.cu", "tracer.cu", "store_reader.cpp", "api.cu"]
HEADERS = ["b2m_common.cuh", "b2m_internal.h", "tile_walker.cuh", "weight_pack.cuh", "fp8_weights.cuh", "int4_weights.cuh",
           "ep_device.cuh", os.path.join("..", "..", "include", "b2m.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-diag-suppress", "177"]
OBJ_DIR = os.path.join(CSRC, "_obj")     # git-ignored (*.o); one object per translation unit, compiled in parallel


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdr_t = max(os.path.getmtime(os.path.join(CSRC, h)) for h in HEADERS if os.path.exists(os.path.join(CSRC, h)))
    procs, objs = [], []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        obj = os.path.join(OBJ_DIR, src + ".o")
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(sp), hdr_t):
            continue
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", sp, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    errs = []
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            errs.append(f"---- {src}\n{out}")
    if errs:
        raise RuntimeError("nvcc failed:\n" + "\n".join(errs))
    cmd = [_nvcc()] + NVCC_FLAGS[:2] + ["-shared", "-o", LIB_PATH] + objs
    if verbose:
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc link failed:\n" + res.stdout + res.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
