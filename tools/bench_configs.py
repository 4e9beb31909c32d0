#!/usr/bin/env python
"""Secondary measurements for the BASELINE.json configs that are not the headline bench line
(bench.py prints the headline line; this script writes the secondary configurations to --out).

  prefill  : Mixtral-8x7B, T = 8*2048 = 16384 tokens through ONE MoE layer (tensor-core bound), TFLOP/s
  offload  : Mixtral-8x7B shapes, reduced depth, half of the experts HBM-resident (config 3 in miniature:
             device_memory_ratio 0.25 of a 180 GB part = 127/256 experts), decode T=8 with on-demand fetch,
             with and without activation-aware prefetch; H2D GB/s, hit rate
  deepseek : DeepSeek-V2-Lite shapes (E=64, k=6, I=1408, 2 shared experts), decode T=16 and prefill T=4096
  h2d      : pinned host -> device copy bandwidth (the roofline of the offload config)
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "moe-infinity_b200")):
    sys.path.insert(0, p)

import numpy as np
import torch

from moe_infinity_b200 import MoEEngine, _lib as L
from moe_infinity_b200 import memory as M


def ev_time(fn, iters, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def h2d_bw():
    n = 1 << 30
    h = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    ms = ev_time(lambda: d.copy_(h, non_blocking=True), 5)
    return n / ms / 1e6


def prefill(T=16384):
    H, I, E, k = 4096, 14336, 8, 2
    eng = MoEEngine(num_layers=1, num_experts=E, hidden=H, inter=I, top_k=k, dtype=torch.bfloat16, max_tokens=T,
                    num_slots=E)
    for e in range(E):
        eng.load_expert(0, e).normal_(0, 0.02)
    eng.set_gate(0, torch.randn(E, H, device="cuda") * 0.02)
    x = torch.randn(T, H, device="cuda").to(torch.bfloat16)
    out = torch.empty_like(x)
    ms = ev_time(lambda: eng.forward(0, x, out=out), 5)
    flops = T * k * 6 * H * I
    st = torch.cuda.current_stream()
    parts = {}
    for name, fn in (("route", lambda: eng.route(0, x)), ("up", lambda: eng.run_experts(0, T, 1)),
                     ("down", lambda: eng.run_experts(0, T, 2)), ("combine", lambda: eng.combine(0, x, out=out))):
        parts[name] = ev_time(fn, 3, warm=1)
    del eng
    return {"T": T, "ms_per_layer": ms, "tflops": flops / ms / 1e9, "parts_ms": parts,
            "flops_per_layer": flops}


def deepseek(T, iters=20):
    Hh, I, E, k, Lr = 2048, 1408, 64, 6, 26
    eng = MoEEngine(num_layers=Lr, num_experts=E, hidden=Hh, inter=I, top_k=k, dtype=torch.bfloat16,
                    expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I,
                    max_tokens=T, num_slots=Lr * E)
    for l in range(Lr):
        for e in range(E):
            eng.load_expert(l, e).normal_(0, 0.02)
        eng.set_gate(l, torch.randn(E, Hh, device="cuda") * 0.05)
        p = C_void()
        eng._ck(eng.lib.b2m_shared_dev_ptr(eng._h, l, p.ref()))
        from moe_infinity_b200.engine import _view
        _view(p.value(), (3 * Hh * 2 * I,), torch.bfloat16, eng.device).normal_(0, 0.02)
        eng._ck(eng.lib.b2m_register_shared(eng._h, l, None, 0))
    x = torch.randn(Lr, T, Hh, device="cuda").to(torch.bfloat16)
    out = torch.empty_like(x)

    def step():
        for l in range(Lr):
            eng.forward(l, x[l], out=out[l])
    step()
    torch.cuda.synchronize()
    counts = []
    for l in range(Lr):
        eng.route(l, x[l])
        counts.append(int((eng.ws("counts", T) > 0).sum()))
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        step()
    ms = ev_time(g.replay, iters)
    expert_b = 3 * Hh * I * 2
    bytes_step = sum(a * expert_b for a in counts) + Lr * 3 * Hh * 2 * I * 2
    flops = Lr * T * (k + 2) * 6 * Hh * I
    del eng
    return {"T": T, "layers": Lr, "ms_per_step": ms, "tokens_per_s": T / ms * 1e3, "avg_active_experts": float(np.mean(counts)),
            "algorithmic_bytes": bytes_step, "hbm_gbs": bytes_step / ms / 1e6, "tflops": flops / ms / 1e9}


def torch_gpu_reference(layers=4, T=8, iters=20):
    """R-torch-gpu (BASELINE.md §4.3): what plain HF-style PyTorch gives on the same GPU for the same path --
    softmax/topk + per-expert index/matmul loop + index_add, ATen/cuBLAS kernels, eager launches.  Written out here
    (not the oracle): this is a measurement of the library path the reference itself calls on the GPU
    (core/parallel/expert_module.cpp:171-175 via torch::matmul), without its offload engine."""
    import torch.nn.functional as F
    H, I, E, k = 4096, 14336, 8, 2
    dev = "cuda"
    w = [[(torch.randn(I, H, device=dev) * 0.02).bfloat16(), (torch.randn(H, I, device=dev) * 0.02).bfloat16(),
          (torch.randn(I, H, device=dev) * 0.02).bfloat16()] for _ in range(E * layers)]
    gates = [(torch.randn(E, H, device=dev) * 0.02).bfloat16() for _ in range(layers)]
    x = torch.randn(layers, T, H, device=dev).bfloat16()

    def step():
        outs = []
        for l in range(layers):
            h = x[l]
            logits = F.linear(h, gates[l])
            p = F.softmax(logits, dim=1, dtype=torch.float)
            pw, sel = torch.topk(p, k, dim=-1)
            pw = (pw / pw.sum(-1, keepdim=True)).to(h.dtype)
            final = torch.zeros_like(h)
            mask = F.one_hot(sel, num_classes=E).permute(2, 1, 0)
            for e in range(E):
                idx, top = torch.where(mask[e])
                if top.numel() == 0:
                    continue
                w1, w2, w3 = w[l * E + e]
                cur = h[top]
                y = F.linear(F.silu(F.linear(cur, w1)) * F.linear(cur, w3), w2)
                final.index_add_(0, top, y * pw[top, idx, None])
            outs.append(final)
        return outs
    ms = ev_time(step, iters, warm=3)
    return {"layers": layers, "T": T, "ms_per_layer": ms / layers, "ms_per_step_32_layers": ms / layers * 32,
            "tokens_per_s_32_layers": T / (ms / layers * 32) * 1e3,
            "note": "eager PyTorch (cuBLAS + ATen), torch.where forces a host sync per expert like the reference"}


class C_void:
    def __init__(self):
        import ctypes
        self.p = ctypes.c_void_p()

    def ref(self):
        import ctypes
        return ctypes.byref(self.p)

    def value(self):
        return self.p.value


def offload(layers=8, steps=24, prefetch=True, resident_frac=127 / 256, skew=1.0):
    H, I, E, k, T = 4096, 14336, 8, 2, 8
    nslots = max(E, int(layers * E * resident_frac))
    eng = MoEEngine(num_layers=layers, num_experts=E, hidden=H, inter=I, top_k=k, dtype=torch.bfloat16,
                    max_tokens=16, num_slots=nslots, max_inflight_prefetch=2)
    t0 = time.perf_counter()
    proto = (torch.randn(3 * H * I) * 0.02).to(torch.bfloat16)
    for l in range(layers):
        for e in range(E):
            blob = torch.empty(3 * H * I, dtype=torch.bfloat16, pin_memory=True)
            blob.copy_(proto)
            blob[:1024] += l + e
            eng._blobs[(l, e)] = blob
            import ctypes as C
            eng._ck(eng.lib.b2m_register_expert(eng._h, l, e, C.c_void_p(blob.data_ptr()), blob.numel() * 2))
    pin_s = time.perf_counter() - t0
    torch.manual_seed(0)
    # skewed, sticky routing (SURVEY §8d): Zipf bias per layer + slowly varying hidden states
    gates, bias = [], []
    for l in range(layers):
        gates.append(torch.randn(E, H, device="cuda") * 0.02)
        eng.set_gate(l, gates[-1])
        perm = torch.randperm(E)
        bias.append((-skew * torch.log(torch.arange(1, E + 1).float()))[perm].cuda())
    x = torch.randn(layers, T, H, device="cuda")
    tracer = M.ExpertTracer(64, layers, E)
    pred = M.ExpertPredictor(layers, E)
    pred.add_tracer(tracer)
    pf = M.ExpertPrefetcher(layers, E)
    pf.set_archer_engine(eng)
    # trace library from the same generator (what load_trace would provide)
    lib = np.zeros((16, layers, E), dtype=np.float32)
    for l in range(layers):
        p = torch.softmax(bias[l].cpu(), 0).numpy()
        lib[:, l, :] = p * 32
    tracer.load_trace(lib)
    seq = tracer.create_entry()
    out = torch.empty(T, H, device="cuda", dtype=torch.bfloat16)
    times = []
    for step in range(steps + 4):
        if step == 4:
            s0 = eng.stats()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        x = 0.9 * x + 0.44 * torch.randn_like(x)
        for l in range(layers):
            xb = x[l].to(torch.bfloat16)
            logits = (xb.float() @ gates[l].t() + bias[l]).to(torch.bfloat16)
            eng.forward(l, xb, router_logits=logits, out=out)
            if prefetch:
                idx = eng.ws("topk_idx", T).cpu().numpy()
                m = pred.predict(seq, idx, l)
                m[l] = 0
                pf.prefetch_experts(l, m)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    s1 = eng.stats()
    d = {k2: s1[k2] - s0[k2] for k2 in s1 if k2 not in ("slots", "slot_bytes", "resident")}
    res = {"layers": layers, "slots": nslots, "experts": layers * E, "prefetch": prefetch, "steps": steps,
           "ms_per_step": wall / steps * 1e3, "ms_per_step_scaled_to_32_layers": wall / steps * 1e3 * 32 / layers,
           "tokens_per_s_scaled_to_32_layers": T / (wall / steps * 32 / layers),
           "hit_rate": d["hits"] / max(1, d["dispatches"]), "misses_per_step": d["misses"] / steps,
           "h2d_gb_per_step": d["h2d_bytes"] / steps / 1e9, "h2d_gbs_achieved": d["h2d_bytes"] / wall / 1e9,
           "prefetch_issued": d["prefetch_issued"], "prefetch_useful": d["prefetch_useful"], "evictions": d["evictions"],
           "pin_seconds": pin_s}
    eng.prefetch_drain()
    del eng
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="h2d,torchgpu,prefill,deepseek,offload")
    ap.add_argument("--out", default="configs.json")
    a = ap.parse_args()
    res = {}
    what = a.what.split(",")
    if "h2d" in what:
        res["h2d_pinned_gbs"] = h2d_bw()
        print("h2d", res["h2d_pinned_gbs"], flush=True)
    if "torchgpu" in what:
        res["torch_gpu_reference_mixtral_decode"] = torch_gpu_reference()
        print(res["torch_gpu_reference_mixtral_decode"], flush=True)
    if "prefill" in what:
        res["mixtral_prefill_T16384_one_layer"] = prefill()
        print(res["mixtral_prefill_T16384_one_layer"], flush=True)
    if "deepseek" in what:
        res["deepseek_v2_lite_decode_T16"] = deepseek(16)
        print(res["deepseek_v2_lite_decode_T16"], flush=True)
        res["deepseek_v2_lite_prefill_T4096"] = deepseek(4096, iters=3)
        print(res["deepseek_v2_lite_prefill_T4096"], flush=True)
    if "offload" in what:
        res["mixtral_offload_half_resident_no_prefetch"] = offload(prefetch=False)
        print(res["mixtral_offload_half_resident_no_prefetch"], flush=True)
        res["mixtral_offload_half_resident_prefetch"] = offload(prefetch=True)
        print(res["mixtral_offload_half_resident_prefetch"], flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
