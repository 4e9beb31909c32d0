"""Throughput of routed experts stored as FP8 E4M3 with one scale per output channel (fp8_scales="row"), against the
128x128 block format and bf16, the three builds alternating in one process.

1. bench.py's headline workload (Mixtral-8x7B shapes, T=8, 16 layers x 8 experts resident, bench.py's seeded weights,
   gates and inputs): tok/s and ms/step of a replayed CUDA graph of the step (CUDA events).
2. One Llama 4 Maverick MoE layer (128 experts, top-1, H=5120, I=8192, its bf16 shared expert of the same size): the layer
   replayed as a CUDA graph at T = 1, 8 and 64 (decode) and 4096 (prefill), tok/s and ms per layer call.
Both fp8 builds quantise the same bf16 numbers (quantize_row / quantize_block128).  bf16 runs without the 12-bit packed
copy (pack_weights=False): the fp8 GEMMs read the same tile walk and launch plan.  Prints one JSON line with the card's
name and power limit (read in the same run).  Needs a GPU.

    python tools/fp8_row_scales.py [--rounds 2] [--steps 50]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "moe-infinity_b200"))

import bench  # noqa: E402
from fp8_decode import _graph_step  # noqa: E402

DT = torch.bfloat16
BUILDS = ("bf16", "block128", "row")


def _engine(build, **kw):
    from moe_infinity_b200 import MoEEngine
    if build == "bf16":
        return MoEEngine(dtype=DT, pack_weights=False, **kw)
    return MoEEngine(dtype=DT, expert_dtype=torch.float8_e4m3fn, fp8_scales=build, **kw)


def _fill(eng, build, L, E, H, I, gate_std=0.02):
    """bench.py's weights (slot by slot N(0, 0.02) in (layer, expert) order from torch.manual_seed(0), then the layer's
    gate); the fp8 builds quantise the same bf16 numbers per matrix."""
    from moe_infinity_b200.fp8 import quantize_block128, quantize_row
    quantize = quantize_row if build == "row" else quantize_block128
    shapes = [(I, H), (H, I), (I, H)] if eng.expert_type == 4 else [(I, H), (I, H), (H, I)]
    torch.manual_seed(0)
    for l in range(L):
        for e in range(E):
            if build == "bf16":
                eng.load_expert(l, e).normal_(0.0, 0.02)
                continue
            w = torch.empty(3 * H * I, dtype=DT, device=eng.device).normal_(0.0, 0.02)
            qs, ss, off = [], [], 0
            for shp in shapes:
                q, s = quantize(w[off:off + shp[0] * shp[1]].view(shp))
                qs.append(q)
                ss.append(s)
                off += shp[0] * shp[1]
            eng.load_expert(l, e, qs, scales=ss)
        eng.set_gate(l, (torch.randn(E, H, device=eng.device) * gate_std).to(DT))


def _free(eng):
    eng.close()
    del eng
    torch.cuda.empty_cache()


def headline(build, steps):
    c = bench.MIXTRAL
    L, E, H, I, k, T = bench.RESIDENT_LAYERS_1GPU, c["E"], c["H"], c["I"], c["k"], bench.BATCH
    eng = _engine(build, num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, max_tokens=16, num_slots=L * E)
    _fill(eng, build, L, E, H, I)
    x = torch.randn(L, T, H, device=eng.device).to(DT)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    _free(eng)
    return {"tokens_per_s": T / ms * 1e3, "ms_per_step": ms}


MAVERICK = dict(E=128, k=1, H=5120, I=8192)


def maverick(build, steps, Ts=(1, 8, 64, 4096)):
    from moe_infinity_b200 import _lib as Lb
    E, k, H, I = MAVERICK["E"], MAVERICK["k"], MAVERICK["H"], MAVERICK["I"]
    eng = _engine(build, num_layers=1, num_experts=E, hidden=H, inter=I, top_k=k, expert_type=Lb.EXPERT_DEEPSEEK,
                  router=Lb.ROUTER_LLAMA4, shared_inter=I, max_tokens=max(Ts), num_slots=E)
    _fill(eng, build, 1, E, H, I, gate_std=0.05)
    g = torch.Generator(device="cuda").manual_seed(1)
    eng.register_shared(0, [(torch.randn(I, H, generator=g, device="cuda") * 0.02).to(DT),
                            (torch.randn(I, H, generator=g, device="cuda") * 0.02).to(DT),
                            (torch.randn(H, I, generator=g, device="cuda") * 0.02).to(DT)])
    res = {}
    for T in Ts:
        x = torch.randn(1, T, H, device=eng.device).to(DT)
        out = torch.empty_like(x)
        ms = _graph_step(eng, x, out, 1, steps if T < 4096 else max(5, steps // 5), warmup=3)
        res[f"T{T}"] = {"tokens_per_s": T / ms * 1e3, "ms_per_layer": ms}
    _free(eng)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tools/fp8_row_scales.py measures on the GPU and there is none")
    gpu = bench.gpu_identity(0)
    head = {b: [] for b in BUILDS}
    mav = {b: [] for b in BUILDS}
    for _ in range(args.rounds):
        for b in BUILDS:
            head[b].append(headline(b, args.steps))
        for b in BUILDS:
            mav[b].append(maverick(b, args.steps))
    print(json.dumps({"gpu": gpu, "mixtral_headline_16_layers_T8": head, "llama4_maverick_layer": mav}), flush=True)


if __name__ == "__main__":
    main()
