"""Full-size DeepSeek-V3 MoE layers on one card: routed experts in FP8 E4M3 (128x128 block scales), the V3 router
(ROUTER_DEEPSEEK_V3: sigmoid, correction bias, top-2-sum groups) in the fused routing kernels.

Shapes: H=7168, I=2048, E=256 routed experts top-8, n_group=8 keep 4, routed_scaling_factor 2.5, norm_topk_prob, one bf16
shared expert with I=2048.  11.3 GB of fp8 experts per layer, so four layers are resident.
1. Graph-captured forward of the four layers at T = 1, 8, 32, 64 (decode) and 1024 (prefill): ms per layer and tok/s
   through the four layers (CUDA events over replays).
2. Routing alone (gate/top-k + permute; a graph of 20 routing calls), fused gate (router_in_kind 0) and logits given
   (kind 1), against ROUTER_DEEPSEEK_GROUP (DeepSeek-V2 group-limited softmax) on the same shapes.
Prints one JSON line with the card's name and power limit (read in the same run).  Needs a GPU.

    python tools/deepseek_v3_layer.py [--steps 50] [--layers 4]
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
H, I, E, K, N_GROUP, TOPK_GROUP, SCALE = 7168, 2048, 256, 8, 8, 4, 2.5
DECODE_T, PREFILL_T = (1, 8, 32, 64), 1024


def _engine(router, L, fp8, max_tokens, num_slots):
    from moe_infinity_b200 import MoEEngine, _lib as Lb
    kw = dict(expert_dtype=torch.float8_e4m3fn) if fp8 else {}
    return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, expert_type=Lb.EXPERT_DEEPSEEK,
                     router=router, n_group=N_GROUP, topk_group=TOPK_GROUP, norm_topk_prob=True, routed_scaling_factor=SCALE,
                     shared_inter=I, max_tokens=max_tokens, num_slots=num_slots, gate_dtype=torch.float32, **kw)


def _fill(eng, L, v3):
    """Eight distinct quantised experts per layer, repeated over the 256 slots (the GEMMs' time does not depend on the
    values; every slot is its own memory), a bf16 shared expert, the gate, and for V3 the correction bias."""
    from moe_infinity_b200.fp8 import quantize_block128
    gen = torch.Generator(device="cuda").manual_seed(0)
    for l in range(L):
        protos = []
        for _ in range(8):
            ws = [torch.randn(shp, device="cuda", generator=gen).mul_(0.02) for shp in ((I, H), (I, H), (H, I))]
            protos.append(tuple(zip(*[quantize_block128(w) for w in ws])))
        for e in range(E):
            qs, ss = protos[e % 8]
            eng.load_expert(l, e, qs, scales=ss)
        eng.register_shared(l, [torch.randn(shp, generator=torch.Generator().manual_seed(l)) * 0.02
                                for shp in ((I, H), (I, H), (H, I))])
        eng.set_gate(l, torch.randn(E, H, device="cuda", generator=gen) * (1.0 / H ** 0.5))
        if v3:
            eng.set_gate_bias(l, torch.randn(E, device="cuda", generator=gen) * 0.1)


def _graph_ms(fn, steps, warmup=3):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
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


def layers(L, steps):
    from moe_infinity_b200 import _lib as Lb
    eng = _engine(Lb.ROUTER_DEEPSEEK_V3, L, True, PREFILL_T, L * E)
    _fill(eng, L, True)
    res = {}
    for T in DECODE_T + (PREFILL_T,):
        x = torch.randn(L, T, H, device="cuda").to(DT)
        out = torch.empty_like(x)

        def step():
            for l in range(L):
                eng.forward(l, x[l], out=out[l])
        ms = _graph_ms(step, steps if T < PREFILL_T else max(5, steps // 5))
        res[f"T={T}"] = {"ms_per_layer": ms / L, "tokens_per_s": T / ms * 1e3}
    st = eng.stats()
    assert st["host_syncs"] == 0 and st["resident"] == L * E
    eng.close()
    return res


def routing(steps, reps=20):
    """Routing only: gate/top-k and permute kernels, no experts (one HBM slot, nothing is run)."""
    from moe_infinity_b200 import _lib as Lb
    res = {}
    for name, router in (("deepseek_v3", Lb.ROUTER_DEEPSEEK_V3), ("deepseek_group_v2", Lb.ROUTER_DEEPSEEK_GROUP)):
        eng = _engine(router, 1, False, PREFILL_T, 1)
        gen = torch.Generator(device="cuda").manual_seed(1)
        eng.set_gate(0, torch.randn(E, H, device="cuda", generator=gen) * (1.0 / H ** 0.5))
        if router == Lb.ROUTER_DEEPSEEK_V3:
            eng.set_gate_bias(0, torch.randn(E, device="cuda", generator=gen) * 0.1)
        for T in DECODE_T + (PREFILL_T,):
            x = torch.randn(T, H, device="cuda", generator=gen).to(DT)
            logits = torch.randn(T, E, device="cuda", generator=gen)
            fused = _graph_ms(lambda: [eng.route(0, x) for _ in range(reps)], steps) / reps
            given = _graph_ms(lambda: [eng.route(0, x, router_logits=logits) for _ in range(reps)], steps) / reps
            res.setdefault(f"T={T}", {})[name] = {"fused_gate_us": fused * 1e3, "logits_given_us": given * 1e3}
        eng.close()
    for v in res.values():
        for kind in ("fused_gate_us", "logits_given_us"):
            v[f"v3_over_v2_{kind[:-3]}"] = v["deepseek_v3"][kind] / v["deepseek_group_v2"][kind]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--layers", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device (H100)")
    card = bench.gpu_identity(0)
    out = {"card": card, "shapes": dict(H=H, I=I, E=E, k=K, n_group=N_GROUP, topk_group=TOPK_GROUP, shared_inter=I,
                                         expert_dtype="fp8_e4m3_b128", layers=args.layers),
           "routing": routing(args.steps), "layers": layers(args.layers, args.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
