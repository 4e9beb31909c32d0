"""Build tests/host/_build/libb2m_hostsim.so = the product's csrc/api.cu (unchanged) + fake_kernels.cpp + fake_cudart.cpp.

TEST INFRASTRUCTURE ONLY.  Lets the CPU suite execute the C-ABI layer's host logic (cache policy, waves, prefetch queue,
launch planning, error handling) without a GPU.  nvcc is needed for api.cu (it includes device headers); nothing here is
used by the product, whose library links the real CUDA runtime and refuses to create a context without a GPU."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
CSRC = os.path.join(ROOT, "moe-infinity_b200", "csrc")
OUT = os.path.join(os.path.dirname(HERE), "_build")
SO = os.path.join(OUT, "libb2m_hostsim.so")


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def build() -> str | None:
    nvcc = _nvcc()
    if nvcc is None or shutil.which("g++") is None:
        return None
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "b2m.h")] + \
           [os.path.join(HERE, f) for f in ("fake_kernels.cpp", "fake_cudart.cpp")]
    if os.path.exists(SO) and os.path.getmtime(SO) >= max(os.path.getmtime(s) for s in srcs):
        return SO
    os.makedirs(OUT, exist_ok=True)
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "include")
    inc = ["-I", CSRC, "-I", os.path.join(ROOT, "include"), "-I", cuda_inc]
    api_o, k_o, r_o = (os.path.join(OUT, n) for n in ("api.o", "fake_kernels.o", "fake_cudart.o"))
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-cudart", "none", "-diag-suppress", "177", *inc, "-c", os.path.join(CSRC, "api.cu"), "-o", api_o],
                   check=True, capture_output=True)
    s_o = os.path.join(OUT, "store_reader.o")           # the product's disk-tier reader is host code: compiled as it is
    for src, obj in ((os.path.join(HERE, "fake_kernels.cpp"), k_o), (os.path.join(HERE, "fake_cudart.cpp"), r_o),
                     (os.path.join(CSRC, "store_reader.cpp"), s_o)):
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", *inc, "-c", src, "-o", obj], check=True, capture_output=True)
    # -Bsymbolic: api.o must bind to THIS library's cuda* emulation even when a real libcudart (torch) is already loaded
    subprocess.run(["g++", "-shared", "-Wl,-Bsymbolic", "-o", SO, api_o, k_o, r_o, s_o, "-lpthread"], check=True, capture_output=True)
    return SO


if __name__ == "__main__":
    print(build())
