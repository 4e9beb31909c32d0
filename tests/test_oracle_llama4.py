"""CPU: tests/llama4_oracle.py restates transformers' Llama4TextMoe.  On the fixtures written by
tests/golden/make_golden_llama4.py from the literal block, the oracle's logits, indices, weights and outputs equal HF's bit
for bit (the generator refuses seeds with a logit tie at the k-th place or a chosen sigmoid within one fp32 ulp of a
rounding boundary, so there is nothing to excuse).  Hand-built cases pin the rounding points of the chain."""
from __future__ import annotations

import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import llama4_oracle as O  # noqa: E402
import make_golden_llama4 as G  # noqa: E402


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_reproduces_hf_block(name):
    d = G.load(name)
    out, logits, idx, w = O.llama4_block(d["x"], d["router_w"], d["gate_up"], d["down"], d["k"], d["shared"])
    assert torch.equal(logits, d["logits"])
    assert not O.kth_ties(logits, d["k"]).any()
    assert torch.equal(idx, d["topk_idx"])
    assert torch.equal(w, d["topk_w"])
    assert torch.equal(out, d["out"])
    assert out.dtype == G.DTYPES[d["dtype"]]


def test_fixtures_cover_the_cases():
    got = {(G.load(n)["dtype"], G.load(n)["E"], G.load(n)["k"]) for n in G.CASES}
    assert {("bf16", 16, 1), ("bf16", 128, 1), ("bf16", 16, 4), ("f16", 16, 2)} <= got


def test_k4_fixture_needs_the_single_rounding():
    """On the k = 4 fixture, rounding after every add of the routed sum gives another output: the fixture pins the
    single rounding of routed_out.sum(dim=0)."""
    d = G.load("llama4_e16k4_bf16")
    x, dt = d["x"], torch.bfloat16
    idx, w = O.llama4_route(d["logits"], d["k"])
    y = O.expert_outputs(x, idx, w, d["gate_up"], d["down"])
    s = O.shared_expert(x, *d["shared"])
    order = idx.argsort(dim=1)
    acc = torch.zeros_like(x)
    for j in range(d["k"]):
        acc = acc + y.gather(1, order[:, j, None, None].expand(-1, 1, x.shape[1])).squeeze(1)   # bf16 add: rounded each time
    per_add = s + acc
    assert torch.equal(O.llama4_combine(y, idx, dt, s), d["out"])
    assert not torch.equal(per_add, d["out"])


def test_k2_sum_is_rounded_once():
    """k = 2: the routed outputs are summed first and rounded once, then added to the rounded shared output
    (shared_expert(x).add_(routed sum)), not accumulated one by one onto the shared output."""
    dt = torch.bfloat16
    y = torch.tensor([[[2 ** -8], [2 ** -8]]])          # exact in bf16
    idx = torch.tensor([[3, 1]])
    s = torch.tensor([[1.0]])
    out = O.llama4_combine(y, idx, dt, s)
    assert out.item() == 1.0 + 2 ** -7                   # r = 2^-7 exactly; 1 + 2^-7 is a bf16 value
    # one rounded add per expert onto the shared output: 1 + 2^-8 is a bf16 tie and rounds to 1.0, twice
    chain = s.to(dt)
    for j in (1, 0):
        chain = chain + y[:, j].to(dt)
    assert chain.item() == 1.0 and out.item() != chain.item()
    # the fp32 numerics add the shared output before the only rounding: 1 + 2^-8 + 2^-9 rounds up
    y2 = torch.tensor([[[2 ** -9], [2 ** -9]]])
    assert O.llama4_combine(y2, idx, dt, torch.tensor([[1.0 + 2 ** -9]]), fp32=True).item() == 1.0 + 2 ** -7
    assert O.llama4_combine(y2, idx, dt, torch.tensor([[1.0 + 2 ** -9]])).item() == 1.0   # round(s) = 1.0; r = 2^-8: tie


def test_route_ranks_logits_and_rounds_the_sigmoid():
    dt = torch.bfloat16
    logits = torch.tensor([[0.5, 3.0, 3.0, -1.0], [20.0, 19.0, 18.0, 25.0]], dtype=dt)
    idx, w = O.llama4_route(logits, 2)
    assert idx.tolist() == [[1, 2], [3, 0]]            # tie at 3.0 -> lower index first; ranked by logit
    assert torch.equal(w, torch.sigmoid(logits.gather(1, idx).float()).to(dt).float())
    # 18, 19, 20 and 25 all give sigmoid 1.0 in bf16 (and 20, 25 in fp32): ranking by sigmoid values could not split them
    assert w[1].tolist() == [1.0, 1.0]
    rows = O.scaled_inputs(torch.tensor([[1.5, -3.0]], dtype=dt), torch.tensor([[0.5, 0.25]]))
    assert rows.tolist() == [[[0.75, -1.5], [0.375, -0.75]]] and rows.dtype == dt


def test_sigmoid_boundary_detector():
    dt = torch.bfloat16
    # sigmoid(0) = 0.5 exactly: a bf16 value, not a boundary
    assert not O.sigmoid_near_boundary(torch.tensor([0.0]), dt).any()
    # a logit whose fp32 sigmoid is the fp32 value next to a bf16 midpoint is flagged
    mid = torch.tensor([0.5 + 2 ** -9], dtype=torch.float32)          # halfway between two bf16 values in [0.5, 1)
    lg = torch.log(mid / (1 - mid))
    p = torch.sigmoid(lg)
    assert (p - mid).abs().item() <= 2 ** -22 and O.sigmoid_near_boundary(lg, dt).all()
