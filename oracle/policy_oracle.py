"""Cache / prefetch policy oracle  --  TEST INFRASTRUCTURE ONLY (never imported by the product).

Pure-Python restatement of the expert residency policy the CUDA engine implements in
moe-infinity_b200/csrc/api.cu, which is itself the *explicit* version of the reference's two
(contradicting, SURVEY.md §9 Q4) eviction loops:

  on-demand fetch   core/parallel/expert_dispatcher.cpp:227-266
      miss and `cache_sizes_[gpu] < byte_size` (:228) -> scan experts (expert-major: `for i in experts: for j in
      layers`, :233-252), take the GPU-resident, unlocked node with the smallest incache_visit_count (strict '<': first
      one wins ties), evict exactly that ONE node and refund its bytes (:256-257);
      incache_visit_count += 1 for every dispatched expert (:264), hit = node was on the GPU (:219);
      `cache_sizes_[gpu] -= byte_size` for EVERY dispatched expert, hit or miss (:266) -- the budget is charged for
      hits as well, so it only ever equals the free HBM while the cache fills by misses alone (policy="reference";
      policy="slots" charges nothing for hits and evicts only when no physical slot is free).
      Eviction does not reset incache_visit_count; only clear_expert_cache_counts does (:175-185).
  activation-aware cache (policy="activation_aware"; B2M_CACHE_ACTIVATION_AWARE in include/b2m.h): the cache the reference
      specifies in moe_infinity/memory/expert_priority_score.py:84-172 / expert_cache.py:95-167 (layer-distance decay x
      activation frequency) but never instantiates (model_offload.py:83).  Victim = resident expert with the largest
      expected time to its next use: layers until its layer runs again + L * (1/f - 1), f = moving average (alpha) of
      "activated in a step", float32 arithmetic, layer-major scan, first maximum wins; physical slots are the budget.
  prefetch          core/prefetch/task_scheduler.h:66-79 (ReplaceCacheCandidates: new protected set, queued
      prefetches dropped), task_scheduler.cpp:82-118 (dedupe), :236-317 (evict-to-fit, skipping protected
      candidates and nodes in use).
Explicit choices (documented in DESIGN.md): victims are never experts of the dispatch in flight; a prefetch never
evicts a protected expert (it is dropped instead); an on-demand miss may, as a last resort.

Parity status: pinned for the on-demand path -- tests/golden/policy_ref_trace.json holds hit / resident-set sequences
recorded from the reference's own compiled engine (oracle/_ref/prefetch_op.so driven by tools/ref_engine_harness.py
--mode policy); tests/test_oracle_policy_ref.py demands this oracle reproduce them and
tests/test_gpu_offload.py demands the CUDA engine reproduce the oracle.  The prefetch side (protected candidates,
evict-to-fit) has no reference test and pins our stated policy only.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Set, Tuple

import numpy as np


class CacheOracle:
    def __init__(self, num_layers: int, num_experts: int, num_slots: int, policy: str = "reference"):
        self.L, self.E, self.nslots = num_layers, num_experts, num_slots
        self.policy = policy
        self.budget = num_slots            # cache_sizes_[gpu] in expert units (expert_dispatcher.cpp:52-54)
        self.alpha = np.float32(0.25)
        self.freq = np.full(num_layers * num_experts, 0.5, dtype=np.float32)
        self.cur_layer = 0
        n = num_layers * num_experts
        self.resident = [False] * n
        self.visits = [0] * n
        self.prefetched_unused = [False] * n
        self.free = num_slots
        self.protected: Set[int] = set()
        self.last_active: List[int] = []
        self.stats = dict(dispatches=0, hits=0, misses=0, evictions=0, prefetch_issued=0, prefetch_useful=0)
        self.evicted_log: List[Tuple[int, int]] = []

    def _id(self, layer, expert):
        return layer * self.E + expert

    def _score(self, i: int) -> np.float32:
        l = i // self.E
        d = (l - self.cur_layer) % self.L
        if d <= 0:
            d += self.L
        f = max(self.freq[i], np.float32(0.02))
        return np.float32(d) + np.float32(self.L) * (np.float32(1.0) / f - np.float32(1.0))

    def _victim(self, in_use: Sequence[int], allow_protected: bool) -> int:
        if self.policy == "activation_aware":
            best, best_s = -1, np.float32(-1.0)
            for i in range(self.L * self.E):       # layer-major, strict '>'
                if not self.resident[i] or i in in_use:
                    continue
                if not allow_protected and i in self.protected:
                    continue
                s = self._score(i)
                if s > best_s:
                    best, best_s = i, s
            return best
        best, best_v = -1, 1 << 60
        for e in range(self.E):            # expert-major scan, strict '<'
            for l in range(self.L):
                i = self._id(l, e)
                if not self.resident[i] or i in in_use:
                    continue
                if not allow_protected and i in self.protected:
                    continue
                if self.visits[i] < best_v:
                    best, best_v = i, self.visits[i]
        return best

    def _acquire(self, in_use: Sequence[int], prefetch: bool) -> bool:
        if self.free > 0:
            self.free -= 1
            return True
        v = self._victim(in_use, False)
        if v < 0 and not prefetch:
            v = self._victim(in_use, True)
        if v < 0:
            return False
        self.resident[v] = False
        self.prefetched_unused[v] = False
        self.stats["evictions"] += 1
        self.evicted_log.append((v // self.E, v % self.E))
        return True

    def _acquire_on_demand(self, in_use: Sequence[int]) -> bool:
        """expert_dispatcher.cpp:227-258: budget used up -> evict exactly one victim."""
        if self.free == 0 or (self.policy == "reference" and self.budget < 1):
            v = self._victim(in_use, False)
            if v < 0:
                v = self._victim(in_use, True)
            if v >= 0:
                self.resident[v] = False
                self.prefetched_unused[v] = False
                self.stats["evictions"] += 1
                self.evicted_log.append((v // self.E, v % self.E))
                self.free += 1
                self.budget += 1                                   # :257
            elif self.free == 0:
                return False
        self.free -= 1
        return True

    def dispatch(self, layer: int, experts: Iterable[int]) -> List[Tuple[int, bool]]:
        """One MoE layer call with the given activated experts.  Returns [(expert, hit)] sorted by expert.
        If the active set does not fit next to itself it is processed in waves (csrc/api.cu b2m_run_experts_ex):
        a wave takes every still-to-run expert that is resident or can get a slot without evicting another
        still-to-run expert; finished waves become evictable."""
        active = [self._id(layer, e) for e in sorted(set(experts))]
        self.cur_layer = layer
        act_set = set(experts)
        for e in range(self.E):            # activation average of this layer's experts (api.cu: before the residency pass)
            i = self._id(layer, e)
            self.freq[i] = (np.float32(1.0) - self.alpha) * self.freq[i] + (self.alpha if e in act_set else np.float32(0.0))
        out = []
        remaining = list(active)
        wave: List[int] = []
        while remaining:
            wave = []
            for i in remaining:
                if self.resident[i]:
                    self.stats["hits"] += 1
                    if self.prefetched_unused[i]:
                        self.stats["prefetch_useful"] += 1
                        self.prefetched_unused[i] = False
                    out.append((i % self.E, True))
                else:
                    if not self._acquire_on_demand(remaining):
                        continue
                    self.stats["misses"] += 1
                    self.resident[i] = True
                    out.append((i % self.E, False))
                self.stats["dispatches"] += 1
                self.visits[i] += 1                                # :264
                self.budget -= 1                                   # :266, hit or miss
                wave.append(i)
            if not wave:
                raise RuntimeError("no evictable slot")
            remaining = [i for i in remaining if i not in wave]
        self.last_active = wave
        return sorted(out)

    def replace_cache_candidates(self, pairs: Iterable[Tuple[int, int]]):
        self.protected = {self._id(l, e) for l, e in pairs}

    def prefetch(self, pairs: Sequence[Tuple[int, int]]):
        """Queued prefetches processed in order (the engine after b2m_prefetch_drain)."""
        for l, e in pairs:
            i = self._id(l, e)
            if self.resident[i]:
                continue
            if not self._acquire(self.last_active, True):
                break       # nothing evictable without touching protected experts: rest of the queue is dropped
            self.resident[i] = True
            self.prefetched_unused[i] = True
            self.stats["prefetch_issued"] += 1

    def prefetch_hint(self, pairs: Sequence[Tuple[int, int]], scores: Sequence[float]):
        order = sorted(range(len(pairs)), key=lambda i: -scores[i])   # stable, descending
        ordered = [pairs[i] for i in order]
        self.replace_cache_candidates(ordered)
        self.prefetch(ordered)

    def clear_counts(self):
        self.visits = [0] * len(self.visits)
