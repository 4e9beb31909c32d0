"""Llama 4 MoE layers (router=ROUTER_LLAMA4) on one GPU.

1. The MoE path of Llama-4-Scout-17B-16E (16 experts top-1, H=5120, I=8192, a 8192-wide shared expert; 48 MoE layers) and
   of Llama-4-Maverick-17B-128E (128 experts top-1, same shapes; 24 MoE layers), every expert resident, the fused router
   gate:
     scout bf16       as many layers as fit (14: 4.3 GB each; without the 12-bit packed copy, which would not fit beside)
     scout int4 bf16  all 48 layers (51.3 GB of routed experts + 12.1 GB of bf16 shared experts)
     scout fp8        24 of the 48 layers
     maverick int4    as many layers as fit (7: 8.6 GB each)
   Decode at T = 1, 8, 64 as a replayed CUDA graph of the step (all layers held): tok/s and ms per layer.  Bytes per step =
   the routed experts the step activates (counted per layer from the routing result) + the shared experts + the router
   weights; their rate as a share of the 3.35 TB/s data-sheet HBM bandwidth.  Prefill at T = 4096, eager, CUDA events.
2. The cost of the Llama 4 routing (logit top-k, rounded sigmoid weights, scaled gather) against the Mixtral routing
   (softmax top-k, plain gather) at E = 16, k = 1, H = 5120, same router weight and inputs, alternating: microseconds per
   routing call (gate + top-k + permute), T = 1, 8, 64, 1024.
Random weights (the cost of these kernels does not depend on the values): one expert's matrices are generated per format
and loaded into every slot.  Prints one JSON line with the card's name and power limit (read in the same run).  Needs a
GPU.

    python tools/llama4_decode.py [--rounds 3] [--steps 30] [--out FILE] [--only NAME,...]
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
H, I = 5120, 8192
CONFIGS = {
    # name: (E, layers, format)
    "scout_bf16": (16, 14, "bf16"),
    "scout_int4_bf16": (16, 48, "int4"),
    "scout_fp8": (16, 24, "fp8"),
    "maverick_int4_bf16": (128, 7, "int4"),
}


def _rnd(g, *shape, std=0.02):
    return (torch.randn(*shape, generator=g, device="cuda") * std).to(torch.bfloat16)


def _engine(E, Ln, fmt, max_tokens=4096):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200 import fp8 as F8
    from moe_infinity_b200 import int4 as I4
    expert_dtype = {"bf16": None, "fp8": torch.float8_e4m3fn, "int4": torch.uint4}[fmt]
    eng = MoEEngine(num_layers=Ln, num_experts=E, hidden=H, inter=I, top_k=1, dtype=torch.bfloat16,
                    expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_LLAMA4, shared_inter=I, max_tokens=max_tokens,
                    num_slots=Ln * E, expert_dtype=expert_dtype, pack_weights=False)
    g = torch.Generator(device="cuda").manual_seed(0)
    ws = [_rnd(g, I, H), _rnd(g, I, H), _rnd(g, H, I)]
    kw = {}
    if fmt == "fp8":
        ws, sc = zip(*[F8.quantize_block128(w) for w in ws])
        kw = dict(scales=sc)
    elif fmt == "int4":
        ws, sc, zs = zip(*[I4.quantize_g128(w, scale_dtype=torch.bfloat16) for w in ws])
        kw = dict(scales=sc, zeros=zs)
    shared = [_rnd(g, I, H), _rnd(g, I, H), _rnd(g, H, I)]
    for l in range(Ln):
        for e in range(E):
            eng.load_expert(l, e, ws, **kw)
        eng.register_shared(l, shared)
        eng.set_gate(l, _rnd(g, E, H, std=0.5))
    del ws, kw
    torch.cuda.synchronize()
    return eng


def _expert_bytes(fmt):
    from moe_infinity_b200 import fp8 as F8
    from moe_infinity_b200 import int4 as I4
    if fmt == "fp8":
        return F8.expert_blob_bytes(H, I)
    if fmt == "int4":
        return I4.expert_blob_bytes(H, I)
    return 3 * H * I * 2


def _bytes_per_step(eng, E, Ln, fmt, x):
    eb = _expert_bytes(fmt)
    total, active = 0, 0
    for l in range(Ln):
        eng.route(l, x[l])
        n = int((eng.ws("counts", x.shape[1]) > 0).sum())
        active += n
        total += n * eb + 3 * H * I * 2 + E * H * 2
    return total, active / Ln


def _prefill_ms(eng, Ln, T, iters=3):
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


def whole_path(name, steps):
    E, Ln, fmt = CONFIGS[name]
    eng = _engine(E, Ln, fmt)
    res = dict(layers=Ln, experts_gb=round(Ln * E * _expert_bytes(fmt) / 1e9, 2))
    for T in (1, 8, 64):
        x = torch.randn(Ln, T, H, device="cuda").to(torch.bfloat16)
        out = torch.empty_like(x)
        ms = _graph_step(eng, x, out, Ln, steps)
        nbytes, act = _bytes_per_step(eng, E, Ln, fmt, x)
        res[f"T{T}"] = dict(tok_s=round(T / ms * 1e3, 1), ms_per_layer=round(ms / Ln, 4), step_ms=round(ms, 4),
                            bytes_per_step=nbytes, experts_per_layer=round(act, 2),
                            hbm_share=round(nbytes / (ms * 1e-3) / HBM_BPS, 4))
    ms = _prefill_ms(eng, Ln, 4096)
    res["prefill_T4096"] = dict(tok_s=round(4096 / ms * 1e3, 1), ms_per_layer=round(ms / Ln, 4))
    assert eng.stats()["host_syncs"] == 0
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def routing_cost(rounds, iters=200):
    """Microseconds per routing call: ROUTER_LLAMA4 against ROUTER_MIXTRAL at E = 16, k = 1, alternating."""
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    E = 16
    g = torch.Generator(device="cuda").manual_seed(1)
    gate = _rnd(g, E, H, std=0.5)
    engs = {}
    for name, router, et, si in (("llama4", L.ROUTER_LLAMA4, L.EXPERT_DEEPSEEK, 128),
                                 ("mixtral", L.ROUTER_MIXTRAL, L.EXPERT_MIXTRAL, 0)):
        eng = MoEEngine(num_layers=1, num_experts=E, hidden=H, inter=128, top_k=1, dtype=torch.bfloat16, expert_type=et,
                        router=router, shared_inter=si, max_tokens=1024, num_slots=E, pack_weights=False)
        eng.set_gate(0, gate)
        engs[name] = eng
    res = {}
    for T in (1, 8, 64, 1024):
        x = torch.randn(T, H, device="cuda").to(torch.bfloat16)
        for eng in engs.values():
            for _ in range(10):
                eng.route(0, x)
        for _ in range(rounds):
            for name, eng in engs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                for _ in range(iters):
                    eng.route(0, x)
                b.record()
                torch.cuda.synchronize()
                res.setdefault(f"T{T}", {}).setdefault(name, []).append(round(a.elapsed_time(b) / iters * 1e3, 2))
    for eng in engs.values():
        eng.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="", help="comma-separated subset of " + ", ".join(list(CONFIGS) + ["routing"]))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    only = set(args.only.split(",")) if args.only else set(CONFIGS) | {"routing"}
    r = {"card": bench.gpu_identity(), "hbm_bps_datasheet": HBM_BPS}
    for name in CONFIGS:
        r[name] = whole_path(name, args.steps) if name in only else "not measured"
    r["routing_us_per_call_e16_k1"] = routing_cost(args.rounds) if "routing" in only else "not measured"
    line = json.dumps(r)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
