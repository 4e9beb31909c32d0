"""CPU: tests/qwen_moe_oracle.py restates the transformers Qwen2-MoE / Qwen3-MoE sparse blocks.  On the fixtures written by
tests/golden/make_golden_qwen_moe.py from the literal blocks, the oracle's indices equal HF's and its weights and outputs
equal HF's bit for bit, except where HF's own k-term sum of the top-k weights (torch's reduction order, norm_topk_prob)
differs from the selection-order sum by one fp32 ulp: those weights are named and bounded at one fp32 ulp, and only the
tokens they scale may differ, by at most one bf16 ulp.  Tokens with tied probabilities at the k-th choice are compared by
the values chosen (torch.topk does not specify which of equal entries it returns)."""
from __future__ import annotations

import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_golden_qwen_moe as G  # noqa: E402
import qwen_moe_oracle as Q  # noqa: E402


def _ulp(t: torch.Tensor) -> torch.Tensor:
    """Spacing of t's dtype at |t| (fp32 or bf16)."""
    nxt = torch.nextafter(t.abs(), torch.full_like(t, float("inf")))
    return nxt - t.abs()


def _by_expert(idx: torch.Tensor, w: torch.Tensor):
    order = idx.argsort(dim=1)
    return idx.gather(1, order), w.gather(1, order)


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_reproduces_hf_block(name):
    d = G.load(name)
    shared = d.get("shared")
    out, logits, idx, w = Q.qwen_block(d["x"], d["gate_w"], d["gate_up"], d["down"], d["k"], d["norm_topk_prob"],
                                       shared, d.get("shared_gate_w"))
    assert torch.equal(logits, d["logits"])
    # bf16 logits tie often; where the k-th and (k+1)-th probabilities are equal, torch.topk's choice among them is
    # unspecified (the oracle and the engine take the lowest index): those tokens are compared by their chosen values only
    tied = Q.topk_ties(logits, d["k"])
    assert tied.float().mean() <= 0.25, f"{int(tied.sum())} of {tied.numel()} tokens tied"
    p = torch.softmax(logits.float(), dim=-1)
    assert torch.equal(p.gather(1, idx)[tied], p.gather(1, d["topk_idx"])[tied])
    # equal probabilities inside the selection may also come out in either order: compare (expert, weight) pairs by expert
    idx, w = _by_expert(idx, w)
    hidx, hw = _by_expert(d["topk_idx"], d["topk_w"])
    assert torch.equal(idx[~tied], hidx[~tied])
    # weights: equal, or one fp32 ulp where the normalising sums differ in order
    wdiff = (w - hw).abs()
    wdiff[tied] = 0
    off = wdiff != 0
    if off.any():
        assert d["norm_topk_prob"] and d["k"] > 1, f"weights differ without normalisation at {off.nonzero().tolist()}"
        assert (wdiff[off] <= _ulp(hw[off])).all(), wdiff[off]
    tok = off.any(dim=1)
    ok = ~tok & ~tied
    assert torch.equal(out[ok], d["out"][ok])
    if tok.any():
        od = (out[tok].float() - d["out"][tok].float()).abs()
        assert (od <= _ulp(d["out"][tok]).float()).all(), f"tokens {tok.nonzero().flatten().tolist()}"


def test_k1_norm_gives_weight_one():
    d = G.load("qwen2_moe_k1_norm_bf16")
    idx, w = Q.qwen_route(d["logits"], 1, True)
    assert torch.equal(w, torch.ones_like(w)) and torch.equal(d["topk_w"], torch.ones_like(w))


def test_combine_chain_rounds_each_step():
    """The chain's rounding points, on hand-picked bf16 values: round(y) * w rounded, then a rounded add per expert in
    ascending id, then round(g * round(s)) and a rounded add."""
    dt = torch.bfloat16
    y = torch.tensor([[[1.0 + 2 ** -9], [3.0]]])                # fp32, not representable in bf16 -> rounded first
    idx = torch.tensor([[5, 2]])                                # expert 2 is applied first
    w = torch.tensor([[0.3, 0.7]])
    out = Q.qwen_combine(y, idx, w, dt)
    a = (torch.tensor([3.0]).to(dt) * torch.tensor([0.7])).to(dt)
    b = (torch.tensor([1.0 + 2 ** -9]).to(dt) * torch.tensor([0.3])).to(dt)
    assert torch.equal(out.reshape(1), (a + b).reshape(1))
    s = torch.tensor([[0.1234567]])
    g = torch.tensor([0.75], dtype=dt)
    out2 = Q.qwen_combine(y, idx, w, dt, s, g)
    assert torch.equal(out2.reshape(1), ((a + b) + (g * s.to(dt).reshape(1))).reshape(1))
