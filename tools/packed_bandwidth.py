"""Bytes and bandwidth of the decode gate/up GEMM (K3) when it reads the experts' 12-bit packed copy.

Builds bench.py's headline workload (Mixtral-8x7B shapes, T=8, N(0, 0.02) bf16 experts, all resident), lets eager forwards
pack every slot, then times K3 per layer with CUDA events exactly as bench.py does (route, event, gate/up phase, event).
Prints one JSON line: packed and bf16 bytes per step and per K3 launch, and K3's bandwidth counted both ways -- the packed
bytes it really streams and the bf16 bytes it stands for.  If K3 streams packed bytes at the rate the bf16 kernel streams bf16
bytes, the packed figure matches bench.py's bf16 K3 bandwidth; if decoding limits it, the packed figure falls short.

    python tools/packed_bandwidth.py [--layers 16] [--iters 10] [--no-pack]
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

REC_BYTES, TILE_ROWS, TILE_COLS = 128 + 12288, 128, 64   # csrc/weight_pack.cuh


def packed_matrix_bytes(rows, cols):
    return (rows // TILE_ROWS) * (cols // TILE_COLS) * REC_BYTES


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.RESIDENT_LAYERS_1GPU)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--no-pack", action="store_true", help="read the bf16 slots (the reference figure)")
    args = ap.parse_args()
    from moe_infinity_b200 import MoEEngine
    cfg = dict(bench.MIXTRAL, L=args.layers)
    L, E, H, I, k, T = cfg["L"], cfg["E"], cfg["H"], cfg["I"], cfg["k"], bench.BATCH
    dev = torch.device("cuda", 0)
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=torch.bfloat16, max_tokens=16,
                    num_slots=L * E, pack_weights=not args.no_pack)
    torch.manual_seed(0)
    for l in range(L):
        for e in range(E):
            eng.load_expert(l, e).normal_(0.0, 0.02)
        eng.set_gate(l, torch.randn(E, H, device=dev) * 0.02)
    x = torch.randn(L, T, H, device=dev).to(torch.bfloat16)
    out = torch.empty_like(x)
    for _ in range(2):                      # eager: packs every slot
        for l in range(L):
            eng.forward(l, x[l], out=out[l])
    torch.cuda.synchronize()
    counts = []
    for l in range(L):
        eng.route(l, x[l])
        counts.append(eng.ws("counts", T).cpu().tolist())
    active = sum(sum(1 for v in c if v > 0) for c in counts)
    bf16_step, bf16_k3 = bench.algorithmic_bytes(counts, T, cfg)
    tok_k3 = L * (T * k * H * 2 + T * k * I * 2)                   # gathered rows in, intermediate out
    pk_k3 = active * 2 * packed_matrix_bytes(I, H) + tok_k3
    pk_step = bf16_step - active * 3 * H * I * 2 + active * (2 * packed_matrix_bytes(I, H) + packed_matrix_bytes(H, I))
    if args.no_pack:
        pk_k3, pk_step = bf16_k3, bf16_step
    st = torch.cuda.current_stream()
    ms = []
    for it in range(3 + args.iters):
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
    k3_ms = sum(ms) / len(ms)
    peak, peak_src = bench.load_peaks()
    line = {
        "packed": not args.no_pack, "layers": L, "tokens": T, "active_experts_per_step": active,
        "bytes_per_step": {"read": pk_step, "bf16_equivalent": bf16_step},
        "k3": {"avg_launch_ms": k3_ms, "bytes_per_launch": pk_k3 / L, "bf16_bytes_per_launch": bf16_k3 / L,
               "streamed_gbs": pk_k3 / L / (k3_ms * 1e-3) / 1e9, "bf16_equivalent_gbs": bf16_k3 / L / (k3_ms * 1e-3) / 1e9,
               "streamed_frac_of_peak": pk_k3 / L / (k3_ms * 1e-3) / 1e9 / peak},
        "peak_gbs": peak, "peak_source": peak_src, "gpu": bench.gpu_identity(0),
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
