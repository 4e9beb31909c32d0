"""Qwen2-MoE / Qwen3-MoE layers (router=ROUTER_QWEN_MOE) on one GPU.

1. The whole MoE path of Qwen1.5-MoE-A2.7B (24 layers, 60 experts top-4, H=2048, I=1408, a gated 5632-wide shared expert;
   bf16) and of Qwen3-30B-A3B (48 layers, 128 experts top-8, H=2048, I=768; bf16 and fp8), every expert resident, the
   fused router gate.  Decode at T = 1, 8, 32, 64 as a replayed CUDA graph of the step (all layers): tok/s and ms per
   layer.  Bytes per step = the routed experts the step activates (counted per layer from the routing result) + the shared
   experts + the router and shared-gate weights; their rate as a share of the 3.35 TB/s data-sheet HBM bandwidth.
   Prefill at T = 4096, eager, CUDA events.
2. The Qwen2 tail (shared-gate kernel + gated combine) against an ungated shared expert (the DeepSeek combine,
   router=ROUTER_DEEPSEEK_GREEDY) at Qwen1.5-MoE-A2.7B shapes, same weights, alternating: ms per step of the captured
   graph of all layers (both engines without the 12-bit packed copy, which could not be made for both at once).
Random weights (the cost of these kernels does not depend on the values).  Prints one JSON line with the card's name and
power limit (read in the same run).  Needs a GPU.

    python tools/qwen_moe_decode.py [--rounds 3] [--steps 50] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "moe-infinity_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from fp8_decode import _graph_step  # noqa: E402

HBM_BPS = 3.35e12
MODELS = {
    # name: (layers, E, k, H, I, shared I, norm_topk_prob)
    "qwen1.5-moe-a2.7b": (24, 60, 4, 2048, 1408, 5632, False),
    "qwen3-30b-a3b": (48, 128, 8, 2048, 768, 0, True),
}


def _engine(model, fp8=False, router=None, max_tokens=4096, pack_weights=True):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200 import fp8 as F8
    Ln, E, k, H, I, SI, norm = MODELS[model]
    router = L.ROUTER_QWEN_MOE if router is None else router
    eng = MoEEngine(num_layers=Ln, num_experts=E, hidden=H, inter=I, top_k=k, dtype=torch.bfloat16,
                    expert_type=L.EXPERT_DEEPSEEK, router=router, norm_topk_prob=norm, shared_inter=SI,
                    max_tokens=max_tokens, num_slots=Ln * E, gate_dtype=torch.bfloat16,
                    expert_dtype=torch.float8_e4m3fn if fp8 else None, pack_weights=pack_weights)
    g = torch.Generator(device="cuda").manual_seed(0)

    def rnd(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device="cuda") * std).to(torch.bfloat16)

    for l in range(Ln):
        for e in range(E):
            ws = [rnd(I, H), rnd(I, H), rnd(H, I)]
            if fp8:
                ws, sc = zip(*[F8.quantize_block128(w) for w in ws])
                eng.load_expert(l, e, ws, scales=sc)
            else:
                eng.load_expert(l, e, ws)
        if SI:
            eng.register_shared(l, [rnd(SI, H), rnd(SI, H), rnd(H, SI)])
            if router == L.ROUTER_QWEN_MOE:
                eng.set_shared_gate(l, rnd(1, H, std=0.05))
        eng.set_gate(l, rnd(E, H, std=0.5))
    torch.cuda.synchronize()
    return eng


def _bytes_per_step(eng, model, x, fp8):
    """Routed experts each layer activates for inputs x[l] + shared experts + router / shared-gate weights."""
    from moe_infinity_b200 import fp8 as F8
    Ln, E, k, H, I, SI, _ = MODELS[model]
    eb = F8.expert_blob_bytes(H, I) if fp8 else 3 * H * I * 2
    total, active = 0, 0
    for l in range(Ln):
        eng.route(l, x[l])
        n = int((eng.ws("counts", x.shape[1]) > 0).sum())
        active += n
        total += n * eb + E * H * 2 + (3 * H * SI * 2 + H * 2 if SI else 0)
    return total, active / Ln


def _prefill_ms(eng, Ln, T, H, iters=3):
    x = torch.randn(Ln, T, H, device="cuda").to(torch.bfloat16)
    out = torch.empty_like(x)
    for l in range(Ln):
        eng.forward(l, x[l], out=out[l])
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        for l in range(Ln):
            eng.forward(l, x[l], out=out[l])
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def whole_path(model, fp8, steps):
    Ln, E, k, H, I, SI, _ = MODELS[model]
    eng = _engine(model, fp8)
    res = {}
    for T in (1, 8, 32, 64):
        x = torch.randn(Ln, T, H, device="cuda").to(torch.bfloat16)
        out = torch.empty_like(x)
        ms = _graph_step(eng, x, out, Ln, steps)
        nbytes, act = _bytes_per_step(eng, model, x, fp8)
        res[f"T{T}"] = dict(tok_s=round(T / ms * 1e3, 1), ms_per_layer=round(ms / Ln, 4), step_ms=round(ms, 4),
                            bytes_per_step=nbytes, experts_per_layer=round(act, 2),
                            hbm_share=round(nbytes / (ms * 1e-3) / HBM_BPS, 4))
    ms = _prefill_ms(eng, Ln, 4096, H)
    res["prefill_T4096"] = dict(tok_s=round(4096 / ms * 1e3, 1), ms_per_layer=round(ms / Ln, 4))
    assert eng.stats()["host_syncs"] == 0
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def tail_cost(rounds, steps):
    """Qwen2 gated shared expert against the ungated (DeepSeek) combine, same shapes and weights, alternating."""
    from moe_infinity_b200 import _lib as L
    model = "qwen1.5-moe-a2.7b"
    Ln, E, k, H, I, SI, _ = MODELS[model]
    # (without the 12-bit packed copy of the experts: two copies of it would not fit beside each other)
    engs = {"qwen_gated": _engine(model, pack_weights=False),
            "deepseek_ungated": _engine(model, router=L.ROUTER_DEEPSEEK_GREEDY, pack_weights=False)}
    res = {}
    for T in (1, 8, 64):
        x = torch.randn(Ln, T, H, device="cuda").to(torch.bfloat16)
        out = torch.empty_like(x)
        for r in range(rounds):
            for name, eng in engs.items():
                res.setdefault(f"T{T}", {}).setdefault(name, []).append(round(_graph_step(eng, x, out, Ln, steps), 4))
    for eng in engs.values():
        eng.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    r = {"card": bench.gpu_identity(), "hbm_bps_datasheet": HBM_BPS}
    r["qwen1.5-moe-a2.7b_bf16"] = whole_path("qwen1.5-moe-a2.7b", False, args.steps)
    r["qwen3-30b-a3b_fp8"] = whole_path("qwen3-30b-a3b", True, args.steps)
    r["qwen3-30b-a3b_bf16"] = whole_path("qwen3-30b-a3b", False, args.steps)
    r["qwen2_tail_ms_per_step"] = tail_cost(args.rounds, args.steps)
    line = json.dumps(r)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
