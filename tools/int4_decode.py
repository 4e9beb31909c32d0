"""Decode and prefill throughput of routed experts stored as 4-bit integers with a bf16 scale and zero point per 128 inputs,
against fp8 and bf16.

1. bench.py's headline workload (Mixtral-8x7B shapes, T=8, 16 layers x 8 experts resident, bench.py's seeded weights, gates
   and inputs), three builds of the experts alternating in one process: the default bf16 build (12-bit packed copy), fp8
   (quantize_block128) and int4 (quantize_g128), both quantised from the same bf16 weights.  Each build reports tok/s and
   ms/step of a replayed CUDA graph of the step (CUDA events) and the gate/up GEMM (K3) alone timed as bench.py does; int4
   also reports the code and group bytes K3 reads over its time, as a fraction of the 3.35 TB/s data-sheet figure.
2. All 32 Mixtral-8x7B layers resident on one card, int4 against fp8.
3. DeepSeek-V2-Lite shapes (26 MoE layers, 64 experts top-6, 2 bf16 shared experts): decode (T=8) and prefill (T=4096) tok/s,
   int4 against fp8 and bf16.
4. Mixtral-8x22B shapes, all 56 layers x 8 experts resident in int4 (71.9 GB), T=8 tok/s -- only when the card has that
   much HBM free; otherwise "skipped".  Timing only: the codes are random bytes with one fixed scale and zero point.
Prints one JSON line with the card's name and power limit (read in the same run).  Needs a GPU.

    python tools/int4_decode.py [--rounds 2] [--steps 50]
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

DT = torch.bfloat16
DATASHEET_GBS = 3350.0   # H100 SXM HBM3


def _fill(eng, L, E, H, I, fmt, std=0.02, gate_std=0.02, gate_dtype=None):
    """bench.py's weights: slot by slot N(0, std) in (layer, expert) order from torch.manual_seed(0), then the layer's gate.
    fp8 / int4: the same bf16 numbers, quantised per matrix."""
    from moe_infinity_b200.fp8 import quantize_block128
    from moe_infinity_b200.int4 import quantize_g128
    dev = eng.device
    torch.manual_seed(0)
    n = 3 * H * I
    shapes = [(I, H), (H, I), (I, H)] if eng.expert_type == 4 else [(I, H), (I, H), (H, I)]
    for l in range(L):
        for e in range(E):
            if fmt in ("bf16", "packed12"):
                eng.load_expert(l, e).normal_(0.0, std)
                continue
            w = torch.empty(n, dtype=DT, device=dev).normal_(0.0, std)
            mats, off = [], 0
            for shp in shapes:
                mats.append(w[off:off + shp[0] * shp[1]].view(shp))
                off += shp[0] * shp[1]
            if fmt == "fp8":
                qs, ss = zip(*[quantize_block128(m) for m in mats])
                eng.load_expert(l, e, qs, scales=ss)
            else:
                qs, ss, zs = zip(*[quantize_g128(m) for m in mats])
                eng.load_expert(l, e, qs, scales=ss, zeros=zs)
        g = torch.randn(E, H, device=dev) * gate_std
        eng.set_gate(l, g if gate_dtype is None else g.to(gate_dtype))


def _kw(fmt):
    return {"fp8": dict(expert_dtype=torch.float8_e4m3fn), "int4": dict(expert_dtype=torch.uint4)}.get(fmt, {})


def headline(fmt, steps):
    from moe_infinity_b200 import MoEEngine
    cfg = dict(bench.MIXTRAL, L=bench.RESIDENT_LAYERS_1GPU)
    L, E, H, I, k, T = cfg["L"], cfg["E"], cfg["H"], cfg["I"], cfg["k"], bench.BATCH
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, max_tokens=16, num_slots=L * E,
                    **_kw(fmt))
    _fill(eng, L, E, H, I, fmt)
    x = torch.randn(L, T, H, device=eng.device).to(DT)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    k3 = _k3_ms(eng, x, out, L, T)
    res = {"tokens_per_s": T / ms * 1e3, "ms_per_step": ms, "k3_avg_launch_ms": k3}
    if fmt == "int4":
        active = 0
        for l in range(L):
            eng.route(l, x[l])
            active += sum(1 for v in eng.ws("counts", T).cpu().tolist() if v > 0)
        per_mat = H * I // 2 + (H * I // 128) * 4                      # codes + group words of one matrix
        k3_bytes = active * 2 * per_mat + L * (T * k * H * 2 + T * k * I * 2)
        gbs = k3_bytes / L / (k3 * 1e-3) / 1e9
        res.update({"active_experts_per_step": active, "k3_bytes_per_launch": k3_bytes / L, "k3_streamed_gbs": gbs,
                    "k3_frac_of_datasheet": gbs / DATASHEET_GBS, "step_weight_bytes": active * 3 * per_mat})
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def full_model(fmt, steps):
    from moe_infinity_b200 import MoEEngine
    c = bench.MIXTRAL
    L, E, H, I, k, T = c["L"], c["E"], c["H"], c["I"], c["k"], bench.BATCH
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, max_tokens=16,
                    device_memory_ratio=0.9, **_kw(fmt))
    _fill(eng, L, E, H, I, fmt)
    x = torch.randn(L, T, H, device=eng.device).to(DT)
    out = torch.empty_like(x)
    st = eng.stats()
    ms = _graph_step(eng, x, out, L, steps)
    st2 = eng.stats()
    res = {"layers": L, "tokens_per_s": T / ms * 1e3, "ms_per_step": ms, "resident": st2["resident"], "slots": st["slots"],
           "slot_bytes": st["slot_bytes"], "misses": st2["misses"]}
    eng.close()
    del eng
    torch.cuda.empty_cache()
    return res


def deepseek(fmt, steps):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as Lb
    Lr, E, H, I, k, Tp = 26, 64, 2048, 1408, 6, 4096
    eng = MoEEngine(num_layers=Lr, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, expert_type=Lb.EXPERT_DEEPSEEK,
                    router=Lb.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I, max_tokens=Tp, num_slots=Lr * E, **_kw(fmt))
    _fill(eng, Lr, E, H, I, fmt, gate_std=0.05, gate_dtype=torch.float32)
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


def mixtral_8x22b(steps):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200.int4 import expert_blob_bytes
    L, E, H, I, k, T = 56, 8, 6144, 16384, 2, bench.BATCH
    need = L * E * expert_blob_bytes(H, I)
    free = torch.cuda.mem_get_info()[0]
    if free < need + (2 << 30):
        return {"skipped": "not enough free HBM", "need_bytes": need, "free_bytes": free}
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, max_tokens=16, num_slots=L * E,
                    expert_dtype=torch.uint4)
    codes = 3 * H * I // 2
    word = (int(torch.tensor(0.004).to(DT).view(torch.int16)) & 0xffff) | (8 << 16)   # s = 0.004, z = 8
    gen = torch.Generator(device="cuda").manual_seed(0)
    for l in range(L):
        for e in range(E):
            v = eng.load_expert(l, e)
            v[:codes].random_(0, 256, generator=gen)
            v[codes:].view(torch.int32).fill_(word)
        eng.set_gate(l, (torch.randn(E, H, device="cuda", generator=gen) * 0.02).to(DT))
    x = torch.randn(L, T, H, device=eng.device).to(DT)
    out = torch.empty_like(x)
    ms = _graph_step(eng, x, out, L, steps)
    st = eng.stats()
    res = {"layers": L, "experts_resident_bytes": need, "tokens_per_s": T / ms * 1e3, "ms_per_step": ms,
           "resident": st["resident"], "misses": st["misses"]}
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
        sys.exit("tools/int4_decode.py measures on the GPU and there is none")
    gpu = bench.gpu_identity(0)
    runs = {"packed12": [], "fp8": [], "int4": []}
    for _ in range(args.rounds):
        for fmt in runs:
            runs[fmt].append(headline(fmt, args.steps))
    full = {"fp8": full_model("fp8", args.steps), "int4": full_model("int4", args.steps)}
    ds = {fmt: deepseek(fmt, args.steps) for fmt in ("bf16", "fp8", "int4")}
    big = mixtral_8x22b(args.steps)
    print(json.dumps({"gpu": gpu, "datasheet_gbs": DATASHEET_GBS, "headline_16_layers_T8": runs,
                      "mixtral_32_layers": full, "deepseek_v2_lite": ds, "mixtral_8x22b_int4_56_layers": big}), flush=True)


if __name__ == "__main__":
    main()
