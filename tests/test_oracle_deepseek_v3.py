"""CPU: the DeepSeek-V3 oracle (tests/deepseek_v3_oracle.py: deepseek_v3_route, deepseek_v3_block) against the fixtures
the literal reference block produced (tests/golden/deepseek_v3_*.pt, tests/golden/make_golden_deepseek_v3.py),
plus hand-built cases for the two places where V3 differs most from V2: masked experts keep choice 0.0 (so with negative
biases they can win), and a single expert is never normalised but always scaled."""
import os

import pytest
import torch

import deepseek_v3_oracle as V3
import make_golden as G
import make_golden_deepseek_v3 as GV3
from oracle import moe_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = sorted(GV3.CASES)


def _load(name):
    fx = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    c = GV3.build(name)
    assert abs(G.checksum([w for e in c["experts"] for w in e]) - fx["weight_checksum"]) < 1e-6 * fx["weight_checksum"]
    assert torch.equal(c["hidden"], fx["hidden"]) and torch.equal(c["gate"], fx["gate"]) and torch.equal(c["bias"], fx["bias"])
    return c, fx


@pytest.mark.parametrize("name", CASES)
def test_v3_route_reproduces_golden(name):
    c, fx = _load(name)
    assert fx["kind"] == "deepseek_v3"
    x = c["hidden"].reshape(-1, c["H"])
    logits = torch.nn.functional.linear(x.float(), c["gate"].float())
    r = V3.deepseek_v3_route(logits, c["bias"], c["k"], c["n_group"], c["topk_group"], c["norm_topk_prob"],
                            c["routed_scaling_factor"])
    assert torch.equal(r.scores, fx["scores"])
    assert torch.equal(r.topk_idx, fx["topk_idx"])
    assert torch.equal(r.topk_weight, fx["topk_weight"])
    r2 = V3.deepseek_v3_route(fx["scores"], c["bias"], c["k"], c["n_group"], c["topk_group"], c["norm_topk_prob"],
                             c["routed_scaling_factor"], are_scores=True)
    assert torch.equal(r2.topk_idx, fx["topk_idx"]) and torch.equal(r2.topk_weight, fx["topk_weight"])


@pytest.mark.parametrize("name", CASES)
def test_v3_block_reproduces_golden(name):
    c, fx = _load(name)
    out, r = GV3.oracle_block(c)
    T = c["B"] * c["S"]
    ok = ~fx["tied"]
    assert bool(ok.all())
    if fx["source"] == "literal":
        assert torch.equal(out.reshape(T, -1)[ok], fx["out"].reshape(T, -1)[ok])
    else:   # the literal block agreed with the oracle to one ulp when the fixture was made; the fixture holds the oracle's
        assert torch.equal(out, fx["out"])


def test_v3_weights_sum_to_the_scale_when_normalised():
    for name in CASES:
        c, fx = _load(name)
        if c["norm_topk_prob"]:
            s = fx["topk_weight"].sum(-1)
            assert torch.allclose(s, torch.full_like(s, c["routed_scaling_factor"]), rtol=1e-6)


def test_masked_expert_with_choice_zero_wins_over_negative_kept_choices():
    """E=8 in 4 groups of 2, topk_group=1, k=2, every bias -1: all choices are negative.  Group 1 (experts 2, 3) has the
    best top-2 sum and is kept; the other six experts are masked to 0.0, which beats every kept (negative) choice.  The
    two winners are the lowest-index masked experts, 0 and 1, and their weights are their UNBIASED sigmoid scores."""
    logits = torch.tensor([[-2.0, -1.5, 3.0, 2.5, -1.0, -3.0, 0.5, -0.5]])
    bias = torch.full((8,), -1.0)
    r = V3.deepseek_v3_route(logits, bias, 2, 4, 1, False, 1.0)
    s = logits.sigmoid()
    choice = s + bias
    assert (choice < 0).all()
    assert r.topk_idx.tolist() == [[0, 1]]
    assert torch.equal(r.topk_weight, s[:, [0, 1]])
    # normalised and scaled: w / (sum + 1e-20) * scale, in selection order
    rn = V3.deepseek_v3_route(logits, bias, 2, 4, 1, True, 2.5)
    w = s[:, [0, 1]]
    assert torch.equal(rn.topk_weight, w / ((w[:, 0] + w[:, 1]).unsqueeze(-1) + 1e-20) * 2.5)
    assert rn.router_mask.tolist() == [[1, 1, 0, 0, 0, 0, 0, 0]]


def test_single_expert_is_scaled_not_normalised():
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(6, 16, generator=g)
    bias = (torch.randn(16, generator=g) * 0.1)
    for norm in (False, True):
        r = V3.deepseek_v3_route(logits, bias, 1, 4, 2, norm, 2.5)
        s = logits.sigmoid()
        assert torch.equal(r.topk_weight, s.gather(1, r.topk_idx) * 2.5)


def test_group_score_is_the_sum_of_the_top_two():
    """One huge choice does not make a group win: the group score is top1 + top2, not the max (V2's rule)."""
    scores = torch.tensor([[0.99, 0.01, 0.80, 0.79]])          # groups {0,1}: 1.00, {2,3}: 1.59
    r = V3.deepseek_v3_route(scores, torch.zeros(4), 2, 2, 1, False, 1.0, are_scores=True)
    assert r.topk_idx.tolist() == [[2, 3]]
    v2 = O.deepseek_route(scores, 2, topk_method="group_limited_greedy", n_group=2, topk_group=1)
    assert v2.topk_idx.tolist() == [[0, 1]]                     # the max rule keeps the other group


def test_literal_reference_gate_matches_oracle():
    """The literal V3 MoEGate on CPU (where the reference tree or its byte-compiled staging exists)."""
    import ref_loader
    if not ref_loader.available():
        pytest.skip("reference tree not present")
    ns = ref_loader.load()
    m = pytest.importorskip("moe_infinity.models.modeling_deepseek_v3", reason="the reference tree has no V3 gate module")
    c = GV3.build("deepseek_v3_norm_bf16")
    gate = m.MoEGate(GV3.config(c)).eval()
    with torch.no_grad():
        gate.weight.copy_(c["gate"].float())
        gate.e_score_correction_bias.copy_(c["bias"])
        idx, w = gate(c["hidden"])
    r = V3.deepseek_v3_route(torch.nn.functional.linear(c["hidden"].reshape(-1, c["H"]).float(), c["gate"].float()),
                            c["bias"], c["k"], c["n_group"], c["topk_group"], True, c["routed_scaling_factor"])
    order = idx.sort(-1)
    assert torch.equal(order.values, r.topk_idx.sort(-1).values)
    ow = torch.gather(w, 1, order.indices)
    rw = torch.gather(r.topk_weight, 1, r.topk_idx.sort(-1).indices)
    assert torch.allclose(ow, rw, rtol=2e-7, atol=0)
    assert ns is not None
