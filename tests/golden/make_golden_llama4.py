"""Generate tests/golden/llama4_*.pt from the LITERAL transformers Llama4TextMoe.

Run:  python tests/golden/make_golden_llama4.py
The block runs on CPU in the case's dtype with seeded weights.  The router is scaled up so that routing is far from
uniform and the sigmoid weights spread over (0, 1).  Each fixture holds x, the router logits (F.linear in the model dtype,
what Llama4Router computes first and returns), the indices and weights the router chose and the block's output.  The
weights are not stored: `weights(name)` regenerates them from the case's seed with torch alone (a checksum in the fixture
guards generator drift).

A seed is refused (generation raises, naming the token) where the result would hang on an unspecified detail rather than
on the spec:
  * a logit tie at the k-th place: torch.topk does not specify which of equal logits it returns;
  * a chosen logit whose fp32 sigmoid lies within one fp32 ulp of a model-dtype rounding boundary: CPU and CUDA compute
    exp differently and may round that weight to different values.
Generation asserts tests/llama4_oracle.py == the literal block, bit for bit.  Only these fixtures are written.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

CASES = {
    # name: (dtype, E, k, H, I, T, seed)
    "llama4_e16k1_bf16": ("bf16", 16, 1, 128, 128, 24, 102),
    "llama4_e128k1_bf16": ("bf16", 128, 1, 128, 128, 16, 102),
    "llama4_e16k4_bf16": ("bf16", 16, 4, 128, 128, 24, 104),
    "llama4_e16k2_f16": ("f16", 16, 2, 128, 128, 24, 104),
}
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}


def path(name: str) -> str:
    return os.path.join(HERE, name + ".pt")


def weights(name: str) -> dict:
    """The case's weights and input, from its seed, in HF's layout: router_w [E,H], gate_up [E,H,2I], down [E,I,H],
    shared (gate [I,H], up [I,H], down [H,I]) and x [T,H]."""
    dt, E, k, H, I, T, seed = CASES[name]
    DT = DTYPES[dt]
    g = torch.Generator().manual_seed(seed)
    w = dict(router_w=(torch.randn(E, H, generator=g) * 0.25).to(DT),           # logits of a few units: weights spread
             gate_up=(torch.randn(E, H, 2 * I, generator=g) * 0.08).to(DT),
             down=(torch.randn(E, I, H, generator=g) * 0.08).to(DT),
             shared=[(torch.randn(I, H, generator=g) * 0.08).to(DT), (torch.randn(I, H, generator=g) * 0.08).to(DT),
                     (torch.randn(H, I, generator=g) * 0.08).to(DT)])
    w["x"] = torch.randn(T, H, generator=g).to(DT)
    return w


def checksum(w: dict) -> float:
    ts = [w["router_w"], w["gate_up"], w["down"], w["x"]] + list(w["shared"])
    return float(sum(t.double().abs().sum() for t in ts))


def make_block(name: str):
    from transformers.models.llama4.configuration_llama4 import Llama4TextConfig
    from transformers.models.llama4.modeling_llama4 import Llama4TextMoe
    dt, E, k, H, I, T, seed = CASES[name]
    cfg = Llama4TextConfig(hidden_size=H, intermediate_size=I, num_local_experts=E, num_experts_per_tok=k,
                           hidden_act="silu")
    w = weights(name)
    blk = Llama4TextMoe(cfg).to(DTYPES[dt]).eval()
    with torch.no_grad():
        blk.router.weight.copy_(w["router_w"])
        blk.experts.gate_up_proj.copy_(w["gate_up"])
        blk.experts.down_proj.copy_(w["down"])
        blk.shared_expert.gate_proj.weight.copy_(w["shared"][0])
        blk.shared_expert.up_proj.weight.copy_(w["shared"][1])
        blk.shared_expert.down_proj.weight.copy_(w["shared"][2])
    return blk, w


def refuse_hazards(name: str, logits: torch.Tensor, idx: torch.Tensor, k: int):
    import llama4_oracle as O
    tied = O.kth_ties(logits, k)
    if tied.any():
        raise ValueError(f"{name}: seed gives a logit tie at the k-th place (tokens {tied.nonzero().flatten().tolist()})")
    near = O.sigmoid_near_boundary(logits.gather(1, idx), logits.dtype)
    if near.any():
        raise ValueError(f"{name}: seed puts a chosen sigmoid within one fp32 ulp of a rounding boundary "
                         f"(tokens {near.any(1).nonzero().flatten().tolist()})")


def generate(name: str) -> dict:
    import llama4_oracle as O
    dt, E, k, H, I, T, seed = CASES[name]
    blk, w_ = make_block(name)
    x = w_["x"]
    with torch.no_grad():
        out, logits = blk(x.unsqueeze(0))
        scores, _ = blk.router(x)
    idx = torch.topk(logits, k, dim=1).indices
    refuse_hazards(name, logits, idx, k)
    topk_w = scores.gather(1, idx).float()
    o_out, o_logits, o_idx, o_w = O.llama4_block(x, w_["router_w"], w_["gate_up"], w_["down"], k, w_["shared"])
    assert torch.equal(o_logits, logits) and torch.equal(o_idx, idx) and torch.equal(o_w, topk_w), name
    assert torch.equal(o_out, out), f"{name}: the oracle differs from the literal block"
    return dict(name=name, dtype=dt, E=E, k=k, H=H, I=I, x=x, logits=logits, topk_idx=idx.to(torch.int64), topk_w=topk_w,
                out=out, checksum=checksum(w_))


def load(name: str) -> dict:
    """The fixture with its weights regenerated (no transformers needed)."""
    d = torch.load(path(name), weights_only=False)
    w = weights(name)
    assert abs(checksum(w) - d["checksum"]) <= 1e-9 * d["checksum"], f"{name}: weight generator drifted"
    d.update(w)
    return d


def main():
    for name in CASES:
        d = generate(name)
        torch.save(d, path(name))
        print("wrote", path(name), os.path.getsize(path(name)), "bytes")


if __name__ == "__main__":
    main()
