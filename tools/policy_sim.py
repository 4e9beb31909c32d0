#!/usr/bin/env python
"""Offline study of BASELINE config 3 (Mixtral-8x7B, device_memory_ratio 0.25 -> 56 of 256 experts resident in 80 GB HBM):
miss counts of cache policies on the SURVEY §8(d) decode trace (per-layer Zipf-skewed gates, sticky hidden states),
computed on the CPU with oracle/policy_oracle.py -- the same policy code the CUDA engine is tested against.

Time model: the step is bound by the host->device link (one Mixtral expert = 352 MB, 6.4 ms at the default --link-gbs 55,
an assumed PCIe Gen5 x16 rate, not a measurement; the MoE math of a step is far shorter), so ms/step ~= misses/step x the
copy time of one expert; a policy can only win by MOVING FEWER BYTES.
  lfu       the reference's on-demand policy (expert_dispatcher.cpp:227-266): evict min incache_visit_count
  belady    clairvoyant optimum (evict the resident expert whose next use is farthest): the floor
  pred:K    lfu + protected set = experts predicted for the next K layers from the previous step's routing of the same
            layer (sticky decoding: what the activation-aware prefetcher can know), no prefetch traffic
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.policy_oracle import CacheOracle  # noqa: E402


def make_trace(L=32, E=8, T=8, k=2, steps=128, skew=1.0, rho=0.9, seed=0, H=256):
    rng = np.random.default_rng(seed)
    gates = rng.standard_normal((L, E, H)).astype(np.float32) / np.sqrt(H)
    bias = np.stack([(-skew * np.log(np.arange(1, E + 1)))[rng.permutation(E)] for _ in range(L)]).astype(np.float32)
    x = rng.standard_normal((L, T, H)).astype(np.float32)
    trace = []
    for s in range(steps):
        x = rho * x + np.sqrt(1 - rho * rho) * rng.standard_normal(x.shape).astype(np.float32)
        for l in range(L):
            logits = x[l] @ gates[l].T + bias[l]
            top = np.argsort(-logits, axis=1, kind="stable")[:, :k]
            trace.append((l, sorted(set(top.flatten().tolist()))))
    return trace


def run_lfu(trace, L, E, slots, protect_next=0):
    orc = CacheOracle(L, E, slots, policy="reference")
    last = {}
    per_layer = len(trace) // (len(trace) // L) if False else L
    for n, (l, act) in enumerate(trace):
        if protect_next:
            cand = []
            for d in range(1, protect_next + 1):
                ll = (l + d) % L
                for e in last.get(ll, []):
                    cand.append((ll, e))
            orc.replace_cache_candidates(cand)
        orc.dispatch(l, act)
        last[l] = act
    return orc.stats


def run_belady(trace, L, E, slots):
    nxt = {}
    next_use = [None] * len(trace)
    for n in range(len(trace) - 1, -1, -1):
        l, act = trace[n]
        next_use[n] = {e: nxt.get((l, e), 1 << 60) for e in act}
        for e in act:
            nxt[(l, e)] = n
    resident = {}
    misses = hits = 0
    for n, (l, act) in enumerate(trace):
        for e in act:
            key = (l, e)
            if key in resident:
                hits += 1
            else:
                misses += 1
                if len(resident) >= slots:
                    cur = {(l, a) for a in act}
                    victim = max((k_ for k_ in resident if k_ not in cur), key=lambda k_: resident[k_])
                    del resident[victim]
            resident[key] = next_use[n][e]
    return {"misses": misses, "hits": hits}


def run_next_use(trace, L, E, slots, alpha=0.25, floor=0.02):
    """Activation-aware eviction: victim = resident expert with the largest EXPECTED time to its next use,
    layer distance (cyclic, decode visits layers in order) + L x (1/f - 1) with f = EMA of 'active in a step'."""
    f = np.full((L, E), 0.5, dtype=np.float64)
    resident = set()
    misses = hits = 0
    for n, (l, act) in enumerate(trace):
        cur = {(l, e) for e in act}
        for e in act:
            if (l, e) in resident:
                hits += 1
                continue
            misses += 1
            if len(resident) >= slots:
                best, best_s = None, -1.0
                for (ll, ee) in resident:
                    if (ll, ee) in cur:
                        continue
                    d = (ll - l) % L
                    if d == 0:
                        d = L
                    sc = d + L * (1.0 / max(f[ll, ee], floor) - 1.0)
                    if sc > best_s:
                        best, best_s = (ll, ee), sc
                resident.discard(best)
            resident.add((l, e))
        a = np.zeros(E)
        a[act] = 1.0
        f[l] = (1 - alpha) * f[l] + alpha * a
    return {"misses": misses, "hits": hits}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--slots", type=int, default=56)
    ap.add_argument("--link-gbs", type=float, default=55.0, help="assumed host->device bandwidth")
    a = ap.parse_args()
    ms_per_miss = 3 * 4096 * 14336 * 2 / (a.link_gbs * 1e9) * 1e3
    L, E = 32, 8
    for skew, rho in ((0.0, 0.0), (1.0, 0.9), (2.0, 0.9), (1.0, 0.99)):
        tr = make_trace(L, E, steps=a.steps, skew=skew, rho=rho)
        warm = L * 16
        trw = tr
        disp = sum(len(x[1]) for x in tr)
        lfu = run_lfu(tr, L, E, a.slots)
        bel = run_belady(tr, L, E, a.slots)
        row = {"lfu": lfu["misses"], "belady": bel["misses"]}
        for K in (4,):
            row[f"pred:{K}"] = run_lfu(tr, L, E, a.slots, protect_next=K)["misses"]
        for al in (0.1, 0.25, 0.5):
            row[f"next:{al}"] = run_next_use(tr, L, E, a.slots, alpha=al)["misses"]
        per_step = {k_: round(v / a.steps, 1) for k_, v in row.items()}
        print(f"skew={skew} rho={rho}: dispatches/step={disp / a.steps:.1f}  misses/step {per_step}  "
              f"-> link-bound ms/step = {{ {', '.join(f'{k_}: {v * ms_per_miss:.0f}' for k_, v in per_step.items())} }}")


if __name__ == "__main__":
    main()
