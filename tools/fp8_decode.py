"""Decode and prefill throughput of routed experts stored as FP8 E4M3 with 128x128 block scales, against bf16.

1. bench.py's headline workload (Mixtral-8x7B shapes, T=8, 16 layers x 8 experts resident, bench.py's seeded weights, gates
   and inputs), three builds of the experts alternating in one process: bf16 slots (pack_weights=False), the 12-bit packed
   copy (default) and fp8 quantised from the same bf16 weights with quantize_block128.  Each build reports tok/s and ms/step
   of a replayed CUDA graph of the step (CUDA events), the gate/up GEMM (K3) alone timed as bench.py does, and, for fp8, the
   bytes K3 streams over its time.
2. All 32 Mixtral layers resident on one card in fp8: tok/s of the full step, resident experts, no offload.
3. DeepSeek-V2-Lite shapes (26 MoE layers, 64 experts top-6, 2 bf16 shared experts): decode (T=8) and prefill (T=4096) tok/s,
   fp8 against bf16.
Prints one JSON line with the card's name and power limit (read in the same run).  Needs a GPU.

    python tools/fp8_decode.py [--rounds 2] [--steps 50]
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

DT = torch.bfloat16


def _fill(eng, L, E, H, I, fp8, std=0.02, gate_std=0.02, gate_dtype=None):
    """bench.py's weights: slot by slot N(0, std) in (layer, expert) order from torch.manual_seed(0), then the layer's gate.
    fp8: the same bf16 numbers, quantised per matrix."""
    from moe_infinity_b200.fp8 import quantize_block128
    dev = eng.device
    torch.manual_seed(0)
    n = 3 * H * I
    for l in range(L):
        for e in range(E):
            if not fp8:
                eng.load_expert(l, e).normal_(0.0, std)
                continue
            w = torch.empty(n, dtype=DT, device=dev).normal_(0.0, std)
            shapes = [(I, H), (H, I), (I, H)] if eng.expert_type == 4 else [(I, H), (I, H), (H, I)]
            qs, ss, off = [], [], 0
            for shp in shapes:
                q, s = quantize_block128(w[off:off + shp[0] * shp[1]].view(shp))
                qs.append(q); ss.append(s)
                off += shp[0] * shp[1]
            eng.load_expert(l, e, qs, scales=ss)
        g = torch.randn(E, H, device=dev) * gate_std
        eng.set_gate(l, g if gate_dtype is None else g.to(gate_dtype))


def _graph_step(eng, x, out, L, steps, warmup=5):
    def step():
        for l in range(L):
            eng.forward(l, x[l], out=out[l])
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        step()
    for _ in range(warmup):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _k3_ms(eng, x, out, L, T, iters=10):
    st = torch.cuda.current_stream()
    ms = []
    for it in range(3 + iters):
        acc = 0.0
        for l in range(L):
            eng.route(l, x[l])
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            eng.run_experts(l, T, phases=1)
            b.record(st)
            eng.run_experts(l, T, phases=2)
            eng.combine(l, x[l], out=out[l])
            b.synchronize()
            acc += a.elapsed_time(b)
        if it >= 3:
            ms.append(acc / L)
    return sum(ms) / len(ms)


def headline(build, steps):
    from moe_infinity_b200 import MoEEngine
    cfg = dict(bench.MIXTRAL, L=bench.RESIDENT_LAYERS_1GPU)
    L, E, H, I, k, T = cfg["L"], cfg["E"], cfg["H"], cfg["I"], cfg["k"], bench.BATCH
    fp8 = build == "fp8"
    kw = dict(expert_dtype=torch.float8_e4m3fn) if fp8 else dict(pack_weights=build == "packed12")
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, max_tokens=16, num_slots=L * E, **kw)
    _fill(eng, L, E, H, I, fp8)
    x = torch.randn(L, T, H, device=eng.device).to(DT)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    k3 = _k3_ms(eng, x, out, L, T)
    res = {"tokens_per_s": T / ms * 1e3, "ms_per_step": ms, "k3_avg_launch_ms": k3}
    if fp8:
        counts = []
        for l in range(L):
            eng.route(l, x[l])
            counts.append(eng.ws("counts", T).cpu().tolist())
        active = sum(sum(1 for v in c if v > 0) for c in counts)
        grid = (I // 128) * (H // 128) * 4
        k3_bytes = active * 2 * (H * I + grid) + L * (T * k * H * 2 + T * k * I * 2)
        res.update({"active_experts_per_step": active, "k3_bytes_per_launch": k3_bytes / L,
                    "k3_streamed_gbs": k3_bytes / L / (k3 * 1e-3) / 1e9,
                    "step_weight_bytes": active * 3 * (H * I + grid)})
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def full_model_fp8(steps):
    from moe_infinity_b200 import MoEEngine
    c = bench.MIXTRAL
    L, E, H, I, k, T = c["L"], c["E"], c["H"], c["I"], c["k"], bench.BATCH
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, max_tokens=16,
                    expert_dtype=torch.float8_e4m3fn, device_memory_ratio=0.9)
    _fill(eng, L, E, H, I, True)
    x = torch.randn(L, T, H, device=eng.device).to(DT)
    out = torch.empty_like(x)
    st = eng.stats()
    ms = _graph_step(eng, x, out, L, steps)
    st2 = eng.stats()
    res = {"layers": L, "tokens_per_s": T / ms * 1e3, "ms_per_step": ms, "resident": st2["resident"], "slots": st["slots"],
           "slot_bytes": st["slot_bytes"], "misses": st2["misses"], "h2d_bytes": st2["h2d_bytes"]}
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def deepseek(fp8, steps):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as Lb
    Lr, E, H, I, k, Tp = 26, 64, 2048, 1408, 6, 4096
    kw = dict(expert_dtype=torch.float8_e4m3fn) if fp8 else {}
    eng = MoEEngine(num_layers=Lr, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, expert_type=Lb.EXPERT_DEEPSEEK,
                    router=Lb.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I, max_tokens=Tp, num_slots=Lr * E, **kw)
    _fill(eng, Lr, E, H, I, fp8, gate_std=0.05, gate_dtype=torch.float32)
    g = torch.Generator(device="cuda").manual_seed(1)
    for l in range(Lr):
        eng.register_shared(l, [(torch.randn(2 * I, H, generator=g, device="cuda") * 0.02).to(DT),
                                (torch.randn(2 * I, H, generator=g, device="cuda") * 0.02).to(DT),
                                (torch.randn(H, 2 * I, generator=g, device="cuda") * 0.02).to(DT)])
    res = {}
    for T, n in ((8, steps), (Tp, max(3, steps // 10))):
        x = torch.randn(Lr, T, H, device=eng.device).to(DT)
        out = torch.empty_like(x)
        ms = _graph_step(eng, x, out, Lr, n, warmup=2)
        res["decode" if T == 8 else "prefill"] = {"T": T, "tokens_per_s": T / ms * 1e3, "ms_per_step": ms}
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tools/fp8_decode.py measures on the GPU and there is none")
    gpu = bench.gpu_identity(0)
    runs = {"bf16": [], "packed12": [], "fp8": []}
    for _ in range(args.rounds):
        for build in runs:
            runs[build].append(headline(build, args.steps))
    full = full_model_fp8(args.steps)
    ds = {"bf16": deepseek(False, args.steps), "fp8": deepseek(True, args.steps)}
    peak, peak_src = bench.load_peaks()
    print(json.dumps({"gpu": gpu, "peak_gbs": peak, "peak_source": peak_src,
                      "headline_16_layers_T8": runs, "mixtral_32_layers_fp8": full, "deepseek_v2_lite": ds}), flush=True)


if __name__ == "__main__":
    main()
