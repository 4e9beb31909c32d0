"""Decode and prefill throughput of int4 experts with fp16 scales and f16 activations (B2M_WEIGHTS_INT4_G128_F16, the AWQ /
GPTQ format) against int4 with bf16 scales and bf16 activations (B2M_WEIGHTS_INT4_G128).  Both decode each value pair with
the same instructions (lop3 / prmt, one x2 subtract, one x2 multiply), so the two should run within noise of each other.

1. bench.py's headline workload (Mixtral-8x7B shapes, T=8, 16 layers x 8 experts resident, bench.py's seeded weights, gates
   and inputs), the two formats alternating in one process, each quantised from the same bf16 weights (quantize_g128 with
   bf16 or fp16 scales).  Each reports tok/s and ms/step of a replayed CUDA graph of the step (CUDA events), the gate/up GEMM
   (K3) alone timed as bench.py does, and the code and group bytes K3 reads per second.
2. All 32 Mixtral-8x7B layers resident on one card, both formats.
3. DeepSeek-V2-Lite shapes (26 MoE layers, 64 experts top-6, 2 shared experts in the activations' type): decode (T=8) and
   prefill (T=4096) tok/s, both formats.
Prints one JSON line with the card's name and power limit (read in the same run).  Needs a GPU.

    python tools/int4_f16_decode.py [--rounds 3] [--steps 50]
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
from fp8_decode import _graph_step, _k3_ms  # noqa: E402

DATASHEET_GBS = 3350.0   # H100 SXM HBM3
DTYPES = {"int4_bf16": torch.bfloat16, "int4_f16": torch.float16}


def _engine(fmt, **kw):
    from moe_infinity_b200 import MoEEngine
    return MoEEngine(dtype=DTYPES[fmt], expert_dtype=torch.uint4, **kw)


def _fill(eng, L, E, H, I, std=0.02, gate_std=0.02, gate_dtype=None):
    """bench.py's weights: slot by slot N(0, std) in bf16, (layer, expert) order from torch.manual_seed(0), quantised per
    matrix with scales of the engine's dtype; then the layer's gate."""
    from moe_infinity_b200.int4 import quantize_g128
    dev = eng.device
    torch.manual_seed(0)
    shapes = [(I, H), (H, I), (I, H)] if eng.expert_type == 4 else [(I, H), (I, H), (H, I)]
    for l in range(L):
        for e in range(E):
            w = torch.empty(3 * H * I, dtype=torch.bfloat16, device=dev).normal_(0.0, std)
            mats, off = [], 0
            for shp in shapes:
                mats.append(w[off:off + shp[0] * shp[1]].view(shp))
                off += shp[0] * shp[1]
            qs, ss, zs = zip(*[quantize_g128(m, scale_dtype=eng.dtype) for m in mats])
            eng.load_expert(l, e, qs, scales=ss, zeros=zs)
        g = torch.randn(E, H, device=dev) * gate_std
        eng.set_gate(l, g.to(gate_dtype or eng.dtype))


def _release(eng):
    eng.close()
    del eng
    torch.cuda.empty_cache()


def headline(fmt, steps):
    cfg = dict(bench.MIXTRAL, L=bench.RESIDENT_LAYERS_1GPU)
    L, E, H, I, k, T = cfg["L"], cfg["E"], cfg["H"], cfg["I"], cfg["k"], bench.BATCH
    eng = _engine(fmt, num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, max_tokens=16, num_slots=L * E)
    _fill(eng, L, E, H, I)
    x = torch.randn(L, T, H, device=eng.device).to(eng.dtype)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    k3 = _k3_ms(eng, x, out, L, T)
    active = 0
    for l in range(L):
        eng.route(l, x[l])
        active += sum(1 for v in eng.ws("counts", T).cpu().tolist() if v > 0)
    per_mat = H * I // 2 + (H * I // 128) * 4                          # codes + group words of one matrix
    k3_bytes = active * 2 * per_mat + L * (T * k * H * 2 + T * k * I * 2)
    gbs = k3_bytes / L / (k3 * 1e-3) / 1e9
    _release(eng)
    return {"tokens_per_s": T / ms * 1e3, "ms_per_step": ms, "k3_avg_launch_ms": k3, "k3_streamed_gbs": gbs,
            "k3_frac_of_datasheet": gbs / DATASHEET_GBS}


def full_model(fmt, steps):
    c = bench.MIXTRAL
    L, E, H, I, k, T = c["L"], c["E"], c["H"], c["I"], c["k"], bench.BATCH
    eng = _engine(fmt, num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, max_tokens=16, device_memory_ratio=0.9)
    _fill(eng, L, E, H, I)
    x = torch.randn(L, T, H, device=eng.device).to(eng.dtype)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    st = eng.stats()
    _release(eng)
    return {"layers": L, "tokens_per_s": T / ms * 1e3, "ms_per_step": ms, "resident": st["resident"], "misses": st["misses"]}


def deepseek(fmt, steps):
    from moe_infinity_b200 import _lib as Lb
    Lr, E, H, I, k, Tp = 26, 64, 2048, 1408, 6, 4096
    eng = _engine(fmt, num_layers=Lr, num_experts=E, hidden=H, inter=I, top_k=k, expert_type=Lb.EXPERT_DEEPSEEK,
                  router=Lb.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I, max_tokens=Tp, num_slots=Lr * E)
    _fill(eng, Lr, E, H, I, gate_std=0.05, gate_dtype=torch.float32)
    g = torch.Generator(device="cuda").manual_seed(1)
    for l in range(Lr):
        eng.register_shared(l, [(torch.randn(2 * I, H, generator=g, device="cuda") * 0.02).to(eng.dtype),
                                (torch.randn(2 * I, H, generator=g, device="cuda") * 0.02).to(eng.dtype),
                                (torch.randn(H, 2 * I, generator=g, device="cuda") * 0.02).to(eng.dtype)])
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
        sys.exit("tools/int4_f16_decode.py measures on the GPU and there is none")
    gpu = bench.gpu_identity(0)
    runs = {fmt: [] for fmt in DTYPES}
    for _ in range(args.rounds):
        for fmt in DTYPES:
            runs[fmt].append(headline(fmt, args.steps))
    full = {fmt: full_model(fmt, args.steps) for fmt in DTYPES}
    ds = {fmt: deepseek(fmt, args.steps) for fmt in DTYPES}
    print(json.dumps({"gpu": gpu, "datasheet_gbs": DATASHEET_GBS, "headline_16_layers_T8": runs,
                      "mixtral_32_layers": full, "deepseek_v2_lite": ds}), flush=True)


if __name__ == "__main__":
    main()
