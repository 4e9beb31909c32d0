"""Pin oracle.moe_oracle.expert_ffn (D1-D3, SURVEY §8a) against the reference's OWN expert modules.

  * test_oracle_matches_reference_golden: always runs; tests/golden/expert_ffn_ref.pt was produced by
    the reference's core/parallel/expert_module.cpp compiled as-is (tests/golden/make_expert_golden.py).
  * test_oracle_matches_live_reference_module: more types, dtypes and shapes, held to SHA-256 digests of the compiled
    reference module's outputs (tests/golden/reference_results.pt, tests/golden/make_ref_golden.py).
Bit equality is demanded: both sides call the same ATen operators.  The recorded outputs were computed on the CPU that
ran the generators, single-threaded; bf16/f16 matmul kernels can differ between CPU types, so on another CPU family a
mismatch here means "regenerate with tests/golden/make_*_golden.py and compare", not necessarily an oracle bug.
"""
from __future__ import annotations

import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import expert_cases as C  # noqa: E402
import make_ref_golden as RG  # noqa: E402
from oracle import moe_oracle as O  # noqa: E402

GOLD = torch.load(os.path.join(HERE, "golden", "expert_ffn_ref.pt"))
REF = torch.load(RG.OUT, weights_only=False)["expert"]


@pytest.mark.parametrize("name", sorted(C.CASES))
def test_oracle_matches_reference_golden(name):
    torch.set_num_threads(1)
    et, di, ws, x = C.make_case(name)
    g = GOLD[name]
    assert abs(sum(float(w.double().abs().sum()) for w in ws) - g["wsum"]) < 1e-9, "weight generator drifted"
    assert torch.equal(x, g["x"])
    y = O.expert_ffn(x, ws, et)
    assert y.dtype == g["y"].dtype and y.shape == g["y"].shape
    assert torch.equal(y, g["y"]), f"{name}: max |diff| {(y.float() - g['y'].float()).abs().max()}"


@pytest.mark.parametrize("et", [0, 1, 2, 3, 4, 5])
@pytest.mark.parametrize("di", [0, 1, 2])
def test_oracle_matches_live_reference_module(et, di):
    torch.set_num_threads(1)
    dt = C.DT[di]
    for i, (H, I, n) in enumerate(RG.EXPERT_SHAPES):
        ws, x = RG.expert_case(et, dt, H, I, n, 1000 + 17 * et + 5 * di + i)
        y = O.expert_ffn(x, ws, et)
        assert RG.digest(y) == REF[(et, di, i)], f"type {et} dtype {dt} shape {(H, I, n)}"


def test_switch_module_casts_weights_to_input_dtype():
    """expert_module.cpp:31-35: fp32 weights, bf16 activations -> weights are cast per call."""
    torch.set_num_threads(1)
    ws, x = RG.expert_case(0, torch.float32, 64, 96, 6, 77)
    assert RG.digest(O.expert_ffn(x.to(torch.bfloat16), ws, 0)) == REF["switch_cast"]
