"""Generate tests/golden/qwen_moe_*.pt from the LITERAL transformers Qwen2MoeSparseMoeBlock / Qwen3MoeSparseMoeBlock.

Run:  python tests/golden/make_golden_qwen_moe.py
The blocks run on CPU in bf16 with seeded weights.  Routers are scaled up so that routing is far from uniform, and the
Qwen2 shared-expert gates so that some gate values round to exactly 0.0 and 1.0.  Each fixture holds x, the router
logits (F.linear in bf16, what the router computes first), the indices and weights HF's router returns and the block's
output.  The weights are not stored: `weights(name)` regenerates them from the case's seed with torch alone (a checksum in
the fixture guards generator drift).  Generation asserts tests/qwen_moe_oracle.py == the literal block (see tests/test_oracle_qwen_moe.py for
the comparison rule).  Only these fixtures are written.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

CASES = {
    # name: (model, E, k, H, I, shared_I, norm_topk_prob, T, seed)
    "qwen2_moe_e60k4_bf16": ("qwen2_moe", 60, 4, 128, 128, 256, False, 24, 71),
    "qwen3_moe_e128k8_bf16": ("qwen3_moe", 128, 8, 128, 128, 0, True, 16, 72),
    "qwen2_moe_k1_norm_bf16": ("qwen2_moe", 16, 1, 128, 128, 128, True, 12, 73),
}
DT = torch.bfloat16


def path(name: str) -> str:
    return os.path.join(HERE, name + ".pt")


def weights(name: str) -> dict:
    """The case's bf16 weights and input, from its seed: gate_w [E,H], gate_up [E,2I,H], down [E,H,I], x [T,H] and, for a
    Qwen2 case, shared (gate, up, down) and shared_gate_w [1,H]."""
    model, E, k, H, I, SI, norm, T, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    w = dict(gate_w=(torch.randn(E, H, generator=g) * 0.25).to(DT),            # scaled router: peaked probabilities
             gate_up=(torch.randn(E, 2 * I, H, generator=g) * 0.08).to(DT),
             down=(torch.randn(E, H, I, generator=g) * 0.08).to(DT))
    if SI:
        w["shared"] = [(torch.randn(SI, H, generator=g) * 0.08).to(DT), (torch.randn(SI, H, generator=g) * 0.08).to(DT),
                       (torch.randn(H, SI, generator=g) * 0.08).to(DT)]
        w["shared_gate_w"] = (torch.randn(1, H, generator=g) * 8.0).to(DT)        # logits of +-90: g rounds to 0.0 / 1.0
    w["x"] = torch.randn(T, H, generator=g).to(DT)
    return w


def checksum(w: dict) -> float:
    ts = [w["gate_w"], w["gate_up"], w["down"], w["x"]] + list(w.get("shared", [])) + \
         ([w["shared_gate_w"]] if "shared_gate_w" in w else [])
    return float(sum(t.double().abs().sum() for t in ts))


def make_block(name: str):
    model, E, k, H, I, SI, norm, T, seed = CASES[name]
    if model == "qwen2_moe":
        from transformers.models.qwen2_moe.configuration_qwen2_moe import Qwen2MoeConfig
        from transformers.models.qwen2_moe.modeling_qwen2_moe import Qwen2MoeSparseMoeBlock
        cfg = Qwen2MoeConfig(hidden_size=H, moe_intermediate_size=I, shared_expert_intermediate_size=SI, num_experts=E,
                             num_experts_per_tok=k, norm_topk_prob=norm, hidden_act="silu")
        blk = Qwen2MoeSparseMoeBlock(cfg)
    else:
        from transformers.models.qwen3_moe.configuration_qwen3_moe import Qwen3MoeConfig
        from transformers.models.qwen3_moe.modeling_qwen3_moe import Qwen3MoeSparseMoeBlock
        cfg = Qwen3MoeConfig(hidden_size=H, moe_intermediate_size=I, num_experts=E, num_experts_per_tok=k,
                             norm_topk_prob=norm, hidden_act="silu")
        blk = Qwen3MoeSparseMoeBlock(cfg)
    w = weights(name)
    blk = blk.to(DT).eval()
    with torch.no_grad():
        blk.gate.weight.copy_(w["gate_w"])
        blk.experts.gate_up_proj.copy_(w["gate_up"])
        blk.experts.down_proj.copy_(w["down"])
        if SI:
            blk.shared_expert.gate_proj.weight.copy_(w["shared"][0])
            blk.shared_expert.up_proj.weight.copy_(w["shared"][1])
            blk.shared_expert.down_proj.weight.copy_(w["shared"][2])
            blk.shared_expert_gate.weight.copy_(w["shared_gate_w"])
    return blk, w


def generate(name: str) -> dict:
    import qwen_moe_oracle as Q
    model, E, k, H, I, SI, norm, T, seed = CASES[name]
    blk, w_ = make_block(name)
    x = w_["x"]
    with torch.no_grad():
        out = blk(x.unsqueeze(0)).squeeze(0)
        logits = torch.nn.functional.linear(x, blk.gate.weight)
        _, w, idx = blk.gate(x)
    d = dict(name=name, model=model, E=E, k=k, H=H, I=I, shared_I=SI, norm_topk_prob=norm, x=x, logits=logits,
             topk_idx=idx.to(torch.int64), topk_w=w.float(), out=out, checksum=checksum(w_))
    if SI:
        gv = Q.shared_gate_values(x, w_["shared_gate_w"])
        assert (gv == 0).any() and (gv == 1).any(), f"{name}: the shared gate values should reach 0.0 and 1.0"
    return d


def load(name: str) -> dict:
    """The fixture with its weights regenerated (no transformers needed)."""
    d = torch.load(path(name), weights_only=False)
    w = weights(name)
    assert abs(checksum(w) - d["checksum"]) <= 1e-9 * d["checksum"], f"{name}: weight generator drifted"
    d.update(w)
    return d


def main():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE)))
    for name in CASES:
        d = generate(name)
        torch.save(d, path(name))
        print("wrote", path(name), os.path.getsize(path(name)), "bytes")


if __name__ == "__main__":
    main()
