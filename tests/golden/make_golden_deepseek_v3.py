"""Generate tests/golden/deepseek_v3_*.pt from the LITERAL reference DeepSeek-V3 block (dev container only).

Run:  python tests/golden/make_golden_deepseek_v3.py
models/deepseek.py's DeepseekMoEBlock with model_type "deepseek_v3" builds the V3 MoEGate (topk_method "noaux_tc", sigmoid
scores, e_score_correction_bias; models/modeling_deepseek_v3/modeling_deepseek.py:436-527) and DeepseekV3MLP experts.  It
runs on CPU with make_golden.py's stand-in executor (the block's own experts, ascending expert id).  Generation asserts
literal == tests/deepseek_v3_oracle.py: bit for bit on untied tokens, or to one output ulp where norm_topk_prob makes the
weights depend on the order torch.topk(sorted=False) returns the experts in.  Only these fixtures are written.
Weights are not stored (regenerated from the seed; a checksum guards generator drift).
"""
from __future__ import annotations

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as G  # noqa: E402  (also puts the repository root and tests/shims on sys.path)
import deepseek_v3_oracle as V3  # noqa: E402
from oracle import moe_oracle as O  # noqa: E402

CASES = {
    # name: (H, I, E, k, n_shared, B, S, dtype, seed, n_group, topk_group, norm, scale)
    "deepseek_v3_norm_bf16": (128, 128, 32, 4, 1, 2, 10, torch.bfloat16, 51, 4, 2, True, 2.5),
    "deepseek_v3_e64k8_bf16": (128, 128, 64, 8, 1, 1, 1, torch.bfloat16, 52, 8, 4, True, 2.5),
    "deepseek_v3_nonorm_bf16": (128, 128, 16, 4, None, 1, 9, torch.bfloat16, 53, 4, 2, False, 1.0),
}


def config(c):
    return types.SimpleNamespace(model_type="deepseek_v3", hidden_size=c["H"], intermediate_size=c["I"] * 4,
                                 moe_intermediate_size=c["I"], n_routed_experts=c["E"], num_experts_per_tok=c["k"],
                                 n_shared_experts=c["n_shared"], routed_scaling_factor=c["routed_scaling_factor"],
                                 scoring_func="sigmoid", seq_aux=False, topk_method="noaux_tc", n_group=c["n_group"],
                                 topk_group=c["topk_group"], norm_topk_prob=c["norm_topk_prob"], hidden_act="silu",
                                 pretraining_tp=1)


def build(name):
    H, I, E, k, ns_, B, S, dtype, seed, n_group, topk_group, norm, scale = CASES[name]
    experts = O.make_experts(E, H, I, dtype, seed, O.DEEPSEEK_MOE_DENSE_ACT_DENSE, std=0.05)
    shared = None
    if ns_ is not None:
        shared = O.make_experts(1, H, I * ns_, dtype, seed + 500, O.DEEPSEEK_MOE_DENSE_ACT_DENSE, std=0.05)[0]
    g = torch.Generator().manual_seed(seed + 3000)
    bias = (torch.randn(E, generator=g) * 0.1).to(torch.bfloat16).float()   # fp32 values representable in bf16
    return dict(H=H, I=I, E=E, k=k, n_shared=ns_, B=B, S=S, dtype=dtype, seed=seed, experts=experts, shared=shared,
                hidden=G.gen_hidden(B, S, H, dtype, seed), gate=G.gen_gate(E, H, dtype, seed, std=2.0), bias=bias,
                n_group=n_group, topk_group=topk_group, norm_topk_prob=norm, routed_scaling_factor=scale)


def run_literal(ns, c):
    blk = ns.deepseek.DeepseekMoEBlock(config(c)).to(c["dtype"])
    blk.eval()                                          # the V3 gate asserts not self.training
    with torch.no_grad():
        blk.gate.weight.copy_(c["gate"])
        blk.gate.e_score_correction_bias.copy_(c["bias"])     # bf16 after .to(dtype): the bias is bf16-representable
        for e in range(c["E"]):
            blk.experts[e].gate_proj.weight.copy_(c["experts"][e][0])
            blk.experts[e].up_proj.weight.copy_(c["experts"][e][1])
            blk.experts[e].down_proj.weight.copy_(c["experts"][e][2])
        if c["n_shared"] is not None:
            blk.shared_experts.gate_proj.weight.copy_(c["shared"][0])
            blk.shared_experts.up_proj.weight.copy_(c["shared"][1])
            blk.shared_experts.down_proj.weight.copy_(c["shared"][2])
    blk.expert_executor = G._StandInExecutor(blk)
    blk.layer_id = 0
    with torch.no_grad():
        return blk(c["hidden"])


def oracle_block(c):
    return V3.deepseek_v3_block(c["hidden"], c["gate"], c["bias"], c["experts"], c["k"], c["shared"], n_group=c["n_group"],
                                topk_group=c["topk_group"], norm_topk_prob=c["norm_topk_prob"],
                                routed_scaling_factor=c["routed_scaling_factor"])


def main():
    import ref_loader
    if not ref_loader.available():
        raise SystemExit("the deepseek_v3 fixtures come from the literal reference block: reference tree absent")
    ns = ref_loader.load()
    for name in CASES:
        c = build(name)
        o_out, r = oracle_block(c)
        l_out = run_literal(ns, c)
        tied = V3.deepseek_v3_choice_ties(r.scores, c["bias"], c["k"], c["n_group"], c["topk_group"])
        T = c["B"] * c["S"]
        lo, oo = l_out.reshape(T, -1), o_out.reshape(T, -1)
        if c["norm_topk_prob"]:
            # the reference sums the k weights in torch.topk(sorted=False) order, the oracle in selection order: the
            # weights are order dependent in the last fp32 bit -> the outputs must agree to one ulp of the output dtype
            ulp = torch.finfo(c["dtype"]).eps
            assert torch.all((lo.float() - oo.float()).abs()[~tied] <= ulp * oo.float().abs()[~tied] + 1e-6), name
            src = "oracle (literal agrees within 1 ulp; topk order dependent)"
        else:
            assert torch.equal(lo[~tied], oo[~tied]), f"{name}: literal != oracle"
            o_out, src = l_out, "literal"
        y32 = O.combine_fp32(c["hidden"], c["experts"], r.topk_idx, r.topk_weight, O.DEEPSEEK_MOE_DENSE_ACT_DENSE,
                             c["shared"])
        torch.save(dict(kind="deepseek_v3", source=src,
                        cfg={k: c[k] for k in ("H", "I", "E", "k", "n_shared", "B", "S", "seed", "n_group", "topk_group",
                                               "norm_topk_prob", "routed_scaling_factor")},
                        dtype=str(c["dtype"]), weight_checksum=G.checksum([w for e in c["experts"] for w in e]),
                        hidden=c["hidden"], gate=c["gate"], bias=c["bias"], scores=r.scores, topk_idx=r.topk_idx,
                        topk_weight=r.topk_weight, tied=tied, out=o_out, out_fp32=y32),
                   os.path.join(HERE, name + ".pt"))
        print(name, src, "ok; untied tokens", int((~tied).sum()), "of", T)


if __name__ == "__main__":
    main()
