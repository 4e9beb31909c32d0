#!/usr/bin/env python
"""Algorithmic bytes / FLOPs and the resulting roofline bounds of the MoE path (SURVEY §8d), from first principles.

  python tools/roofline_model.py                 # the BASELINE configs
  python tools/roofline_model.py --model mixtral --tokens 8 --gpus 8

Decode is HBM bound: per layer the weights of the A *distinct activated* experts are streamed once,
E[A] = E * (1 - (1 - k/E)^T) for uniform routing; prefill is tensor bound: 6*H*I FLOP per (token, expert).
Peaks are NVIDIA's data-sheet figures of the H100 card named by --card (default sxm; a card run below its rated power
reaches less)."""
from __future__ import annotations

import argparse
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = {
    # H, I, E, k, MoE layers, shared I (0 = none), gate bytes per element
    "mixtral": dict(H=4096, I=14336, E=8, k=2, L=32, shared=0, gate_b=2),
    "deepseek_v2_lite": dict(H=2048, I=1408, E=64, k=6, L=26, shared=2816, gate_b=4),
}


PEAKS = {
    "sxm": dict(hbm_gbs=3350.0, bf16_tflops=989.0, source="H100 SXM data sheet (HBM3, dense bf16)"),
    "pcie": dict(hbm_gbs=2000.0, bf16_tflops=756.0, source="H100 PCIe data sheet (HBM2e, dense bf16)"),
    "nvl": dict(hbm_gbs=3900.0, bf16_tflops=835.0, source="H100 NVL data sheet (HBM3, dense bf16)"),
}


def layer(model: dict, T: int, gpus: int = 1):
    H, I, E, k = model["H"], model["I"], model["E"], model["k"]
    expert_bytes = 3 * H * I * 2
    # expert parallel: a rank owns E/gpus experts; the global batch is T*gpus tokens, every rank sees all of it
    Tg = T * gpus
    El = E // gpus
    active = E * (1.0 - (1.0 - k / E) ** Tg) / gpus if gpus > 1 else E * (1.0 - (1.0 - k / E) ** T)
    active = min(active, El)
    w_bytes = active * expert_bytes + (3 * H * model["shared"] * 2 if model["shared"] else 0)
    io_bytes = 2 * T * H * 2 + T * E * model["gate_b"] + T * k * 8
    flops = Tg * k * 6 * H * I / gpus + (T * 6 * H * model["shared"] if model["shared"] else 0)
    return dict(active_experts=active, weight_bytes=w_bytes, io_bytes=io_bytes, bytes=w_bytes + io_bytes, flops=flops,
                expert_bytes=expert_bytes)


def report(name: str, T: int, gpus: int, card: str = "sxm"):
    m, p = MODELS[name], PEAKS[card]
    lay = layer(m, T, gpus)
    L = m["L"]
    t_hbm = lay["bytes"] / (p["hbm_gbs"] * 1e9)
    t_tc = lay["flops"] / (p["bf16_tflops"] * 1e12)
    bound = "hbm" if t_hbm >= t_tc else "tensor"
    t = max(t_hbm, t_tc)
    out = dict(model=name, tokens_per_gpu=T, gpus=gpus, active_experts_per_rank=round(lay["active_experts"], 2),
               bytes_per_layer=lay["bytes"], flops_per_layer=lay["flops"], bytes_per_step=lay["bytes"] * L,
               bound=bound, min_ms_per_layer=t * 1e3, min_ms_per_step=t * L * 1e3,
               max_tokens_per_s=T * gpus / (t * L), peaks=p["source"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=sorted(MODELS))
    ap.add_argument("--tokens", type=int, default=8)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--card", choices=sorted(PEAKS), default="sxm")
    a = ap.parse_args()
    if a.model:
        print(json.dumps(report(a.model, a.tokens, a.gpus, a.card), indent=1))
        return
    rows = [("mixtral", 8, 1), ("mixtral", 8, 2), ("mixtral", 8, 4), ("mixtral", 8, 8), ("mixtral", 16384, 1),
            ("deepseek_v2_lite", 16, 1), ("deepseek_v2_lite", 4096, 1), ("deepseek_v2_lite", 65536, 1)]
    print(f"{'model':18s} {'T/gpu':>6s} {'gpus':>4s} {'A/rank':>7s} {'GB/step':>9s} {'TFLOP/step':>11s} {'bound':>7s} "
          f"{'min ms/step':>12s} {'max tok/s':>11s}")
    for name, T, g in rows:
        r = report(name, T, g, a.card)
        print(f"{name:18s} {T:6d} {g:4d} {r['active_experts_per_rank']:7.2f} {r['bytes_per_step'] / 1e9:9.2f} "
              f"{r['flops_per_layer'] * MODELS[name]['L'] / 1e12:11.2f} {r['bound']:>7s} {r['min_ms_per_step']:12.3f} "
              f"{r['max_tokens_per_s']:11.0f}")


if __name__ == "__main__":
    main()
