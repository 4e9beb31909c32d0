#!/usr/bin/env python
"""Drive the reference's OWN native engine (oracle/_ref/prefetch_op.so) on the GPU box  --  TEST / BASELINE INFRASTRUCTURE.

The "T1" tier of SURVEY §8c / the R-gpu timing of §8d: builds a reduced-L MoE stack, hands its tensors to the reference
engine exactly the way moe_infinity/runtime/model_offload.py does (offload -> register placeholders -> expert_dispatcher
-> set_topology -> register_expert), then per layer performs what `DistributedExpertExecutor.dispatch_local` + the block's
Python combine do (expert_executor.py:32-58, mixtral.py:87-101).

Modes (one reference engine per process: global singletons, archer_prefetch_handle.cpp:18-28 -> run each as a subprocess):
  --mode policy    small experts, HBM budget = --slots experts; replays a seeded trace of (layer, active experts) through
                   the real GPUFetchFunc (expert_dispatcher.cpp:191-307) and records, per dispatched expert, the `hit`
                   flag wait_expert() returns and the resident set afterwards (is_tensor_on_device).  Two protocols:
                   "sequential" = one expert per set_expected_queue(1)/enqueue/wait (deterministic: every earlier expert
                   has been unlocked by OutputFunc, :397-434) and "batch" = dispatch_local's all-at-once enqueue (which
                   experts of the layer are still locked when a later miss scans for a victim depends on thread timing).
                   Output: a JSON trace (committed as tests/golden/policy_ref_trace.json).  Also compares every
                   wait_expert() output with this repository's compat.expert_dispatcher on the same inputs.
  --mode timing    full-size Mixtral experts, --layers deep; ms/layer of the reference engine next to ours.

Gotchas taken from the reference code (SURVEY §8 c.2):
  * >= 2 dense stages per GPU or InitializeTopology divides by zero (model_topology.cpp:518,525);
  * the expert_dispatcher is constructed BEFORE set_topology in the real flow (model_offload.py:471-477 vs :606), which is
    what makes its HBM budget ratio x total memory (expert_dispatcher.cpp:52-54);
  * the offload directory must accept O_DIRECT (archer_aio_utils.cpp:17; tmpfs does not): candidates are probed, and if
    none works the process re-executes itself under oracle/_ref/libnodirect.so (our LD_PRELOAD shim that clears O_DIRECT);
  * any DLOG_FATAL aborts the process; never destroy the engine objects (destructors join threads blocked on condition
    variables) -> os._exit at the end.

  python tools/ref_engine_harness.py --mode policy --out policy_ref_trace.json
  python tools/ref_engine_harness.py --mode timing --layers 4 --tokens 8 --steps 16 --ratio 0.9
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "moe-infinity_b200"))


def load_reference_engine():
    so = os.path.join(ROOT, "oracle", "_ref", "prefetch_op.so")
    if not os.path.exists(so):
        raise SystemExit(f"{so} missing: make -C oracle/ref_build -f Makefile.engine (needs the reference tree)")
    import torch  # noqa: F401  (libtorch first)
    spec = importlib.util.spec_from_file_location("prefetch_op", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _accepts_o_direct(d: str) -> bool:
    try:
        os.makedirs(d, exist_ok=True)
        p = os.path.join(d, ".odirect_probe")
        fd = os.open(p, os.O_RDWR | os.O_CREAT | os.O_DIRECT, 0o660)
        try:
            import mmap
            buf = mmap.mmap(-1, 4096)          # page aligned
            buf.write(b"x" * 4096)
            ok = os.write(fd, buf) == 4096
        finally:
            os.close(fd)
            os.unlink(p)
        return ok
    except OSError:
        return False


def pick_store_dir(want: str, need_bytes: int) -> str:
    """First candidate directory that accepts O_DIRECT and has room; else re-exec under the no-O_DIRECT preload shim."""
    import shutil
    cands = [want, "/var/tmp/b2m_ref_store", "/tmp/b2m_ref_store", "/dev/shm/b2m_ref_store"]
    preload = "libnodirect.so" in os.environ.get("LD_PRELOAD", "")
    for d in cands:
        if not d:
            continue
        try:
            os.makedirs(d, exist_ok=True)
            free = shutil.disk_usage(d).free
        except OSError:
            continue
        if free < need_bytes * 1.1 + (1 << 30):
            continue
        if preload or _accepts_o_direct(d):
            # a fresh store per run: the reference reuses an existing archer_index and aborts on a size mismatch
            # (archer_tensor_handle.cpp:40-50,69-72)
            return tempfile.mkdtemp(prefix="run_", dir=d)
    if not preload:
        shim = os.path.join(ROOT, "oracle", "_ref", "libnodirect.so")
        if os.path.exists(shim):
            env = dict(os.environ, LD_PRELOAD=shim + (":" + os.environ["LD_PRELOAD"] if os.environ.get("LD_PRELOAD") else ""))
            print("[harness] no O_DIRECT-capable directory with room: re-executing under", shim, flush=True)
            os.execve(sys.executable, [sys.executable] + sys.argv, env)
    raise SystemExit("no usable offload directory (O_DIRECT + free space) and no preload shim")


class RefStack:
    """The reference engine loaded with a Mixtral-shaped expert stack, the way model_offload.py loads it."""

    def __init__(self, P, store_dir, ratio, L_, E, H, I, dt, threads, std=0.02, seed=0, keep_host_copy=True):
        import torch
        self.P, self.L, self.E, self.H, self.I, self.dt = P, L_, E, H, I, dt
        # ---- 1. engine + tensor store (one handle per process)
        self.h = P.prefetch_handle(store_dir, ratio)
        g = torch.Generator().manual_seed(seed)
        self.ids, next_id = {}, 0
        dense = []
        for _ in range(2):                                           # two tiny dense stages (see gotchas)
            t = torch.randn(64, 64, generator=g).to(dt)
            self.h.offload(t, next_id)
            dense.append(next_id)
            next_id += 1
        self.experts = {}
        big = H * I > (1 << 22)          # full-size experts: one seeded draw per layer, experts are rescaled copies (CPU randn
        for l in range(L_):              # of 5.6 G values would cost a minute of GPU-box time and changes nothing measured)
            if big:
                base = [torch.randn(I, H, generator=g) * std, torch.randn(H, I, generator=g) * std, torch.randn(I, H, generator=g) * std]
            for e in range(E):
                if big:
                    ws = [(b * (1.0 + 0.03 * e)).to(dt) for b in base]
                else:
                    ws = [(torch.randn(I, H, generator=g) * std).to(dt), (torch.randn(H, I, generator=g) * std).to(dt),
                          (torch.randn(I, H, generator=g) * std).to(dt)]          # w1, w2, w3 (expert_module.cpp:139-145)
                if keep_host_copy:
                    self.experts[(l, e)] = ws
                self.ids[(l, e)] = list(range(next_id, next_id + 3))
                for t, tid in zip(ws, self.ids[(l, e)]):
                    self.h.offload(t, tid)                                          # model_offload.py:894-899
                next_id += 3
        self.placeholders = {}
        for tid in range(next_id):
            self.placeholders[tid] = torch.zeros(1, dtype=dt)                      # model_offload.py:755,764
            self.h.register(self.placeholders[tid], tid)
        # ---- 2. dispatcher first, then the topology (real order), then expert registration
        self.d = P.expert_dispatcher(E, L_, 0, 4, threads)                         # dtype 0 = bf16, type 4 = Mixtral
        topology = [(f"dense{i}", [[dense[i]]]) for i in range(2)]
        topology += [(f"layer{l}", [self.ids[(l, e)] for e in range(E)]) for l in range(L_)]
        self.h.set_topology(topology)                                              # model_offload.py:767-768
        for (l, e), t in self.ids.items():
            self.d.register_expert(l, e, t)                                        # :851-853

    def resident(self):
        return sorted([l, e] for (l, e), t in self.ids.items() if self.h.is_tensor_on_device(int(t[0])))


def make_trace(L_, E, steps, seed):
    """Seeded (layer, active experts) requests: skewed so that the cache has something to keep."""
    import numpy as np
    rng = np.random.default_rng(seed)
    pop = np.array([1.0 / (r + 1) for r in range(E)])
    trace = []
    for s in range(steps):
        for l in range(L_):
            perm = np.roll(np.arange(E), l)                       # each layer has its own popular experts
            p = pop[np.argsort(perm)]
            n = int(rng.integers(2, 5))
            act = sorted(rng.choice(E, size=n, replace=False, p=p / p.sum()).tolist())
            trace.append({"step": s, "layer": l, "experts": act})
    return trace


def mode_policy(args):
    import torch
    L_, E, H, I = args.layers, args.experts, args.hidden, args.inter
    dt = torch.bfloat16
    expert_bytes = 3 * H * I * 2
    assert (H * I * 2) % 4096 == 0, "tensor sizes must be multiples of the 4 KiB aio alignment (model_topology.cpp:429-431)"
    total = torch.cuda.mem_get_info(0)[1]                         # == GetTotalDeviceMemory (cuda_utils.cpp:33-38)
    ratio = (args.slots + 0.5) * expert_bytes / total             # cache_sizes_ = ratio x total (expert_dispatcher.cpp:52-54)
    store = pick_store_dir(args.dir, L_ * E * expert_bytes)
    P = load_reference_engine()
    ref = RefStack(P, store, ratio, L_, E, H, I, dt, args.threads, std=0.05, seed=args.seed)
    budget_experts = int(ratio * total) // expert_bytes
    assert budget_experts == args.slots, (budget_experts, args.slots)
    trace = make_trace(L_, E, args.steps, args.seed)
    T = args.tokens
    g = torch.Generator().manual_seed(args.seed + 1)
    xs = [torch.randn(T, H, generator=g).to(dt).cuda() for _ in range(L_)]

    def mask_for(active):
        m = torch.zeros(T, E, dtype=torch.bool)
        for t in range(T):
            m[t, active[t % len(active)]] = True
            m[t, active[(t + 1) % len(active)]] = True
        return m.cuda()

    # compare wait_expert() outputs with this repository's dispatcher on the same inputs (same weights, same masks)
    from moe_infinity_b200 import compat
    oh = compat.prefetch_handle(os.path.join(store, "ours_unused"), 0.0)
    tid = 0
    our_ids = {}
    for (l, e), ws in ref.experts.items():
        our_ids[(l, e)] = list(range(tid, tid + 3))
        for w, i in zip(ws, our_ids[(l, e)]):
            oh.offload(w, i)
        tid += 3
    od = compat.expert_dispatcher(E, L_, 0, 4, args.threads, handle=oh, top_k=2, max_tokens=max(T, 16), num_slots=args.slots)
    for (l, e), t in our_ids.items():
        od.register_expert(l, e, t)

    out = {"config": {"layers": L_, "experts": E, "hidden": H, "inter": I, "slots": args.slots, "tokens": T, "seed": args.seed,
                      "steps": args.steps, "ratio": ratio, "expert_bytes": expert_bytes, "total_mem": total,
                      "engine": "reference prefetch_op.so (core/parallel/expert_dispatcher.cpp GPUFetchFunc)"},
           "trace": trace, "sequential": [], "batch": [], "clear_counts_at": []}
    worst_rel, n_cmp, n_bit = 0.0, 0, 0
    ours_hits_equal = True
    half = len(trace) // 2
    # ---- protocol 1: sequential (deterministic)
    for n, req in enumerate(trace):
        l, act = req["layer"], req["experts"]
        if n == half:                                              # pin clear_expert_cache_counts too (:175-185)
            ref.d.clear_expert_cache_counts()
            od.clear_expert_cache_counts()
            out["clear_counts_at"].append(n)
        mask = mask_for(act)
        for e in act:
            ref.d.set_inputs(xs[l], mask)
            ref.d.set_expected_queue(1)
            ref.d.enqueue_expert(l, e, 0, False)
            res = ref.d.wait_expert()
            assert len(res) == 1
            y, rl, re_, hit = res[0]
            assert (rl, re_) == (l, e)
            out["sequential"].append({"n": n, "layer": l, "expert": e, "hit": int(hit), "resident_after": ref.resident()})
            od.set_inputs(xs[l], mask)
            od.set_expected_queue(1)
            od.enqueue_expert(l, e, 0, False)
            ores = od.wait_expert()
            oy, _, _, ohit = ores[0]
            torch.cuda.synchronize()
            ours_hits_equal &= int(ohit) == int(hit)
            yf, of = y.float(), oy.float()
            rms = yf.pow(2).mean().sqrt().item()
            worst_rel = max(worst_rel, (yf - of).abs().max().item() / max(rms, 1e-9))
            n_cmp += yf.numel()
            n_bit += int((y == oy).sum().item())
    out["outputs_vs_ours"] = {"max_abs_diff_over_rms": worst_rel, "frac_bit_identical": n_bit / max(n_cmp, 1),
                              "hit_flags_equal": bool(ours_hits_equal), "elements": n_cmp}
    ours_res = sorted([l, e] for (l, e) in our_ids if od.engine.is_resident(l, e))
    out["outputs_vs_ours"]["resident_set_equal_at_end"] = ours_res == ref.resident()
    out["resident_after_sequential"] = ref.resident()
    # ---- protocol 2: batch (dispatch_local's all-at-once enqueue), continuing from the state above; run twice over the
    # trace to see whether thread timing changes the outcome
    for rep in range(2):
        for n, req in enumerate(trace):
            l, act = req["layer"], req["experts"]
            mask = mask_for(act)
            ref.d.set_inputs(xs[l], mask)
            ref.d.set_expected_queue(len(act))
            for e in act:
                ref.d.enqueue_expert(l, e, 0, False)
            res = ref.d.wait_expert()
            hits = {int(e): int(h) for _, _, e, h in res}
            out["batch"].append({"rep": rep, "n": n, "layer": l, "hits": [hits[e] for e in act], "resident_after": ref.resident()})
    path = args.out or "policy_ref_trace.json"
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f)
    print(json.dumps({"mode": "policy", "out": path, "dispatches": len(out["sequential"]),
                      "hits": sum(r["hit"] for r in out["sequential"]), **out["outputs_vs_ours"]}), flush=True)
    import shutil
    shutil.rmtree(store, ignore_errors=True)
    os._exit(0)


def mode_timing(args):
    import torch
    import torch.nn.functional as F
    L_, E, H, I, k, T = args.layers, args.experts, args.hidden, args.inter, args.top_k, args.tokens
    dt = torch.bfloat16
    expert_bytes = 3 * H * I * 2
    store = pick_store_dir(args.dir, L_ * E * expert_bytes)
    P = load_reference_engine()
    if args.budget_experts > 0:                                   # forced offload: HBM budget of N experts
        args.ratio = (args.budget_experts + 0.5) * expert_bytes / torch.cuda.mem_get_info(0)[1]
    t0 = time.perf_counter()
    ref = RefStack(P, store, args.ratio, L_, E, H, I, dt, args.threads, std=0.02, seed=0, keep_host_copy=bool(args.compare))
    setup_s = time.perf_counter() - t0
    d = ref.d
    g = torch.Generator().manual_seed(1)
    gates = [(torch.randn(E, H, generator=g) * 0.05).to(dt).cuda() for _ in range(L_)]
    xs = [torch.randn(T, H, generator=g).to(dt).cuda() for _ in range(L_)]
    hits = [0, 0]

    def ref_layer(l, x):
        """mixtral.py:44-101 with dispatch_local (expert_executor.py:32-58) on the reference engine"""
        logits = F.linear(x, gates[l])
        rw = F.softmax(logits, dim=1, dtype=torch.float)
        rw, sel = torch.topk(rw, k, dim=-1)
        rw = (rw / rw.sum(dim=-1, keepdim=True)).to(x.dtype)
        mask = F.one_hot(sel, num_classes=E)
        wmask = (rw[..., None] * mask).permute(0, 2, 1).sum(dim=-1)
        mask = mask.permute(0, 2, 1).sum(dim=-1).to(torch.bool)
        count = mask.sum(dim=0).cpu().numpy().flatten()                            # the reference's per-layer host sync
        active = [e for e in range(E) if count[e] > 0]
        out = torch.zeros_like(x)
        if args.protocol == "batch":                                               # dispatch_local: all at once
            d.set_inputs(x, mask)
            d.set_expected_queue(len(active))
            for e in active:
                d.enqueue_expert(l, e, 0, False)
            results = d.wait_expert()
        else:
            # one expert per enqueue/wait.  Needed whenever the engine evicts: GPUFetchFunc's victim scan try_locks EVERY
            # node (expert_dispatcher.cpp:239-245) while the Python thread is still enqueueing the layer's other experts,
            # whose own try_lock then fails -> DLOG_FATAL -> abort (:127-132).  Observed with 352 MB experts
            # the single fetch thread serialises the copies anyway.
            results = []
            for e in active:
                d.set_inputs(x, mask)
                d.set_expected_queue(1)
                d.enqueue_expert(l, e, 0, False)
                results += d.wait_expert()
        for y, _, e, hit in results:
            idx = mask[:, e]
            out[idx] += y.to(x.device) * wmask[idx, e][:, None]
            hits[1] += 1
            hits[0] += int(hit)
        return out, logits

    def run_ref():
        return [ref_layer(l, xs[l]) for l in range(L_)]

    for _ in range(args.warmup):
        run_ref()
    torch.cuda.synchronize()
    hits[0] = hits[1] = 0
    per_step = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        outs = run_ref()
        torch.cuda.synchronize()
        per_step.append((time.perf_counter() - t0) * 1e3)
    ref_ms = sum(per_step) / len(per_step)
    res = {"mode": "timing", "impl": "reference native engine (prefetch_op.so)", "layers": L_, "tokens": T, "ratio": args.ratio,
           "hidden": H, "inter": I, "experts": E, "setup_s": setup_s, "budget_experts": args.budget_experts, "store_dir": store,
           "ms_per_step": ref_ms, "ms_per_step_median": sorted(per_step)[len(per_step) // 2], "ms_per_layer": ref_ms / L_,
           "tokens_per_s_32_layers": T / (ref_ms / L_ * 32 / 1e3), "hit_rate": hits[0] / max(hits[1], 1),
           "resident_experts": len(ref.resident()), "threads": args.threads, "protocol": args.protocol,
           "h2d_gb_per_step": (1.0 - hits[0] / max(hits[1], 1)) * hits[1] / max(args.steps, 1) * expert_bytes / 1e9}

    # ---- this repository's engine on the same weights and the reference's own router logits
    if args.compare:
        from moe_infinity_b200 import MoEEngine
        eng = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dt, max_tokens=max(T, 16),
                        num_slots=L_ * E)
        for (l, e), ws in ref.experts.items():
            eng.load_expert(l, e, ws)
        for l in range(L_):
            eng.set_gate(l, gates[l])
        worst = 0.0
        for l in range(L_):
            ref_out, logits = outs[l]
            ours = eng.forward(l, xs[l], router_logits=logits)
            torch.cuda.synchronize()
            rms = ref_out.float().pow(2).mean().sqrt().item()
            worst = max(worst, (ours.float() - ref_out.float()).abs().max().item() / max(rms, 1e-9))
        for _ in range(3):
            for l in range(L_):
                eng.forward(l, xs[l])
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.steps):
            for l in range(L_):
                eng.forward(l, xs[l])
        ev1.record()
        torch.cuda.synchronize()
        ours_ms = ev0.elapsed_time(ev1) / args.steps
        res.update({"ours_ms_per_step": ours_ms, "ours_ms_per_layer": ours_ms / L_, "speedup": ref_ms / ours_ms,
                    "max_abs_diff_over_rms": worst})
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f)
    import shutil
    shutil.rmtree(store, ignore_errors=True)
    os._exit(0)            # never run the reference's destructors (see gotchas)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["policy", "timing"], default="timing")
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--experts", type=int, default=8)
    ap.add_argument("--hidden", type=int, default=None)
    ap.add_argument("--inter", type=int, default=None)
    ap.add_argument("--top-k", type=int, default=2)
    ap.add_argument("--tokens", type=int, default=8)
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--slots", type=int, default=9, help="policy mode: HBM budget in experts")
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--ratio", type=float, default=0.9, help="timing mode: device_memory_ratio handed to prefetch_handle")
    ap.add_argument("--dir", default="")
    ap.add_argument("--out", default="")
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--budget-experts", type=int, default=0, help="timing mode: derive --ratio from an HBM budget of N experts")
    ap.add_argument("--protocol", choices=["batch", "sequential"], default="batch",
                    help="timing mode: dispatch_local's all-at-once enqueue, or one expert per enqueue/wait (forced offload)")
    ap.add_argument("--compare", type=int, default=1, help="timing mode: also run this repo's engine and compare hidden states")
    args = ap.parse_args()
    if args.mode == "policy":
        args.layers = args.layers or 3
        args.hidden = args.hidden or 256
        args.inter = args.inter or 512
        args.steps = args.steps or 10
        mode_policy(args)
    else:
        args.layers = args.layers or 4
        args.hidden = args.hidden or 4096
        args.inter = args.inter or 14336
        args.steps = args.steps or 8
        mode_timing(args)


if __name__ == "__main__":
    main()
