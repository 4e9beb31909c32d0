"""Cost of act-order GPTQ experts (B2M_WEIGHTS_INT4_G128_F16 with a b2m_set_input_perm table per layer) against the same
format in natural order.  The only new device work is the gather in the routing kernels: each gathered row reads its
expert's table row and the token's row element by element instead of copying 16-byte vectors.

1. Routing alone, Mixtral-8x7B shapes (H=4096, E=8, top-2), T = 1, 8, 64, 1024: a CUDA graph of 20 routing calls (fused
   gate, top-k, permute and gather), with and without a table, in microseconds per call (CUDA events).
2. bench.py's headline shape (16 Mixtral-8x7B layers resident, T=8, tools/int4_f16_decode.py's weights) with and without a
   table per layer, alternating in one process: tok/s of a replayed graph of the step.
3. DeepSeek-V2-Lite shapes (26 MoE layers, 64 experts top-6, f16 shared experts): decode (T=8) and prefill (T=4096), with
   and without tables.
The tables are random permutations: what the gather costs does not depend on the weights.  Prints one JSON line with the
card's name and power limit (read in the same run).  Needs a GPU.

    python tools/int4_act_order.py [--rounds 3] [--steps 50]
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
from int4_f16_decode import _engine, _fill, _release  # noqa: E402

MODES = ("natural", "act_order")


def _tables(eng, layers, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for l in layers:
        eng.set_input_perm(l, torch.stack([torch.randperm(eng.H, generator=g, device="cuda") for _ in range(eng.E)]))


def routing(rounds, calls=20, reps=50):
    c = bench.MIXTRAL
    H, E, k = c["H"], c["E"], c["k"]
    eng = _engine("int4_f16", num_layers=1, num_experts=E, hidden=H, inter=c["I"], top_k=k, max_tokens=1024, num_slots=1)
    eng.set_gate(0, (torch.randn(E, H, device="cuda") * 0.02).to(torch.float16))
    table = torch.stack([torch.randperm(H, device="cuda") for _ in range(E)])
    res = {m: {} for m in MODES}
    for T in (1, 8, 64, 1024):
        x = torch.randn(T, H, device="cuda").to(torch.float16)
        graphs = {}
        for m in MODES:
            eng.set_input_perm(0, table if m == "act_order" else None)
            for _ in range(2):
                eng.route(0, x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(calls):
                    eng.route(0, x)
            graphs[m] = g
        for _ in range(rounds):
            for m in MODES:
                graphs[m].replay()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                for _ in range(reps):
                    graphs[m].replay()
                b.record()
                b.synchronize()
                res[m].setdefault(f"T{T}", []).append(a.elapsed_time(b) * 1e3 / (reps * calls))
    _release(eng)
    return res


def headline(mode, steps):
    cfg = dict(bench.MIXTRAL, L=bench.RESIDENT_LAYERS_1GPU)
    L, E, H, I, k, T = cfg["L"], cfg["E"], cfg["H"], cfg["I"], cfg["k"], bench.BATCH
    eng = _engine("int4_f16", num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, max_tokens=16, num_slots=L * E)
    _fill(eng, L, E, H, I)
    if mode == "act_order":
        _tables(eng, range(L))
    x = torch.randn(L, T, H, device=eng.device).to(eng.dtype)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    _release(eng)
    return {"tokens_per_s": T / ms * 1e3, "ms_per_step": ms}


def deepseek(mode, steps):
    from moe_infinity_b200 import _lib as Lb
    Lr, E, H, I, k, Tp = 26, 64, 2048, 1408, 6, 4096
    eng = _engine("int4_f16", num_layers=Lr, num_experts=E, hidden=H, inter=I, top_k=k, expert_type=Lb.EXPERT_DEEPSEEK,
                  router=Lb.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I, max_tokens=Tp, num_slots=Lr * E)
    _fill(eng, Lr, E, H, I, gate_std=0.05, gate_dtype=torch.float32)
    g = torch.Generator(device="cuda").manual_seed(1)
    for l in range(Lr):
        eng.register_shared(l, [(torch.randn(2 * I, H, generator=g, device="cuda") * 0.02).to(eng.dtype),
                                (torch.randn(2 * I, H, generator=g, device="cuda") * 0.02).to(eng.dtype),
                                (torch.randn(H, 2 * I, generator=g, device="cuda") * 0.02).to(eng.dtype)])
    if mode == "act_order":
        _tables(eng, range(Lr))
    res = {}
    for T, n in ((8, steps), (Tp, max(3, steps // 10))):
        x = torch.randn(Lr, T, H, device=eng.device).to(eng.dtype)
        out = torch.empty_like(x)
        ms = _graph_step(eng, x, out, Lr, n, warmup=2)
        res["decode" if T == 8 else "prefill"] = {"T": T, "tokens_per_s": T / ms * 1e3, "ms_per_step": ms}
    _release(eng)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tools/int4_act_order.py measures on the GPU and there is none")
    gpu = bench.gpu_identity(0)
    route = routing(args.rounds)
    head = {m: [] for m in MODES}
    ds = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for m in MODES:
            head[m].append(headline(m, args.steps))
    for _ in range(max(1, args.rounds - 1)):
        for m in MODES:
            ds[m].append(deepseek(m, args.steps))
    print(json.dumps({"gpu": gpu, "routing_us_per_call": route, "headline_16_layers_T8": head, "deepseek_v2_lite": ds}),
          flush=True)


if __name__ == "__main__":
    main()
