#!/usr/bin/env python
"""Compile the reference's hot-path PYTHON files for the GPU box  --  TEST INFRASTRUCTURE ONLY.

The Python half of the reference is built the same way as its C++ half (oracle/ref_build/Makefile*): compiled from the
sources where they lie under $REF, outputs only into oracle/_ref/ (git-ignored, travels to the GPU box with the
snapshot).  For Python "compiled" means byte-compiled: every hot-path module becomes a sourceless `<module>.pyc` under
oracle/_ref/pyref/, which `tests/shims/ref_loader.py` imports where /root/reference does not exist, so that the
reference's own unmodified blocks can be executed on the GPU on top of this repository's `compat` objects
(tests/test_gpu_literal_blocks.py).  No reference source text is copied anywhere; the product package never reads
oracle/_ref/.

  python oracle/ref_build/stage_pyref.py            # needs /root/reference (dev container only)
"""
from __future__ import annotations

import os
import py_compile
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "_ref", "pyref")
REF = os.environ.get("B2M_REFERENCE_ROOT", "/root/reference")
# hot-path files only (SURVEY §2 rows 1, 3, 4 + the vendored DeepSeek-V2 gate the DeepSeek block imports, row 2)
FILES = [
    "moe_infinity/models/mixtral.py",
    "moe_infinity/models/deepseek.py",
    "moe_infinity/models/switch_transformers.py",
    "moe_infinity/models/nllb_moe.py",
    "moe_infinity/models/modeling_deepseek/__init__.py",
    "moe_infinity/models/modeling_deepseek/modeling_deepseek.py",
    "moe_infinity/models/modeling_deepseek/configuration_deepseek.py",
    "moe_infinity/models/modeling_deepseek/tokenization_deepseek_fast.py",   # imported by the package __init__
    "moe_infinity/distributed/expert_executor.py",
    "moe_infinity/memory/__init__.py",
    "moe_infinity/memory/expert_tracer.py",
    "moe_infinity/memory/expert_predictor.py",
    "moe_infinity/memory/expert_prefetcher.py",
    "moe_infinity/memory/expert_entry.py",
    "moe_infinity/memory/expert_cache.py",
    "moe_infinity/memory/expert_priority_score.py",
    "moe_infinity/utils/config.py",
    "moe_infinity/utils/hf_config.py",
    "moe_infinity/utils/__init__.py",
    "moe_infinity/common/constants.py",
]


def stage(verbose: bool = True) -> str | None:
    if not os.path.isdir(os.path.join(REF, "moe_infinity")):
        return None
    n = 0
    for rel in FILES:
        src = os.path.join(REF, rel)
        if not os.path.exists(src):
            continue
        dst = os.path.join(OUT, rel) + "c"          # sourceless layout: <module>.pyc next to where the .py would be
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not os.path.exists(dst) or os.path.getmtime(dst) < os.path.getmtime(src):
            py_compile.compile(src, cfile=dst, dfile=rel, doraise=True)
        n += 1
    if verbose:
        print(f"byte-compiled {n} reference python modules into {OUT}")
    return OUT


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
