"""Activation-aware expert tracing / prediction / prefetch request building (host policy, P1-P4).

Mirrors the reference's moe_infinity/memory/{expert_tracer,expert_predictor,expert_prefetcher}.py
(same class and method names, same results) with two changes that matter on the GPU:
  * no device round trips: the reference keeps the trace library on cuda:0 and pays two host syncs per
    sequence per layer (expert_tracer.py:104,120,124); here the library is a NumPy array on the host and
    `find_most_similar` is one vectorised expression (the library is <= 1000 x L x E floats);
  * the prefetcher hands (layer, expert, score) triples to the C-ABI scheduler in ONE call
    (b2m_prefetch_hint) instead of a Python loop of replace_cache_candidates + enqueue_prefetch
    (memory/expert_prefetcher.py:42-59).
The arithmetic follows the reference line by line so tests/test_memory_policy.py can demand equality with
the literal reference classes.
"""
from __future__ import annotations

import copy
import os
import uuid
from collections import Counter
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np


@dataclass
class ExpertTraceEntry:  # memory/expert_entry.py:6-14
    seq_id: str = None
    matrix: np.ndarray = None
    access: int = 0
    num_new_tokens: int = 0

    def __hash__(self):
        return hash(self.seq_id)


class ExpertTracer:
    """expert_tracer.py:17-125.  `num_layers`/`num_experts` replace parse_moe_param(config)."""

    def __init__(self, capacity: int, num_layers: int, num_experts: int, num_encoder_layers: int = 0):
        self.num_layers, self.num_experts, self.num_encoder_layers = num_layers, num_experts, num_encoder_layers
        self.capacity = capacity
        self.trace: Dict[str, ExpertTraceEntry] = {}
        self.trace_collection = np.zeros((capacity, num_layers, num_experts), dtype=np.float32)  # :33-35
        self.collection_access = np.zeros((capacity,))
        self.persistent_capacity = 0

    def load_trace(self, trace: Union[os.PathLike, str, np.ndarray]):  # :40-52 (also accepts str, see SURVEY Q9)
        if isinstance(trace, (os.PathLike, str)):
            trace = np.load(trace, allow_pickle=False)
        trace = np.asarray(trace, dtype=np.float32)
        n = trace.shape[0]
        assert n <= self.capacity, (f"loaded trace capacity {n} must be less than or equal to capacity in config "
                                    f"{self.capacity}")
        self.trace_collection[:n] = trace
        self.persistent_capacity = n

    def create_entry(self) -> str:  # :54-59
        seq_id = uuid.uuid4().hex
        self.trace[seq_id] = ExpertTraceEntry(seq_id, np.zeros((self.num_layers, self.num_experts)), 0, 0)
        return seq_id

    def finish_entry(self, seq_id):  # :61-76 (intent of the reference; its version mixes numpy/torch)
        trace_sum = self.trace_collection.sum(axis=(1, 2))
        if np.any(trace_sum == 0):
            idx = int(np.argwhere(trace_sum == 0)[0][0])
        else:
            acc = self.collection_access.copy()
            acc[: self.persistent_capacity] = 1e9
            idx = int(np.argmin(acc))
        self.trace_collection[idx] = self.trace[seq_id].matrix
        self.collection_access[idx] = 1

    def update_entry(self, seq_id, expert_list, layer_idx):  # :78-84
        counter = Counter(np.asarray(expert_list).flatten().tolist())
        for key, count in counter.items():
            self.trace[seq_id].matrix[layer_idx, key] += count
        if layer_idx == self.num_layers - 1:
            self.trace[seq_id].num_new_tokens += 1

    def get_entry_decoder(self, seq_id):  # :86-89
        entry = copy.deepcopy(self.trace[seq_id])
        entry.matrix[: self.num_encoder_layers, :] = 0
        return entry

    def get_entry(self, seq_id):
        return self.trace[seq_id]

    def find_most_similar(self, matrix: np.ndarray, layer_idx: int) -> np.ndarray:  # :94-125
        lib = self.trace_collection.copy()
        lib[:, : (layer_idx + 1), :] = 1e-9
        with np.errstate(divide="ignore", invalid="ignore"):
            lib = lib / lib.sum(axis=2, keepdims=True)
            m = matrix.astype(np.float64).copy()
            m = (m / m.sum(axis=1, keepdims=True)).astype(np.float32)
        m = np.nan_to_num(m)
        # nn.CosineSimilarity(dim=2, eps=1e-6): x.y / (max(|x|,eps) * max(|y|,eps))
        num = (m[None] * lib).sum(axis=2)
        den = np.maximum(np.linalg.norm(m, axis=1), 1e-6)[None] * np.maximum(np.linalg.norm(lib, axis=2), 1e-6)
        with np.errstate(invalid="ignore"):
            cos_dist = 1 - (num / den).mean(axis=1)
        # torch.argmin treats NaN as the minimum and returns the first one
        nan = np.isnan(cos_dist)
        min_idx = int(np.argmax(nan)) if nan.any() else int(np.argmin(cos_dist))
        self.collection_access[min_idx] += 1
        return self.trace_collection[min_idx].copy()


class ExpertPredictor:
    """expert_predictor.py:7-35."""

    def __init__(self, num_layers: int, num_experts: int, num_encoder_layers: int = 0):
        self.num_layers, self.num_experts, self.num_encoder_layers = num_layers, num_experts, num_encoder_layers
        self.layer_decay_func = lambda x, l, L: -1 / (L + 1) * (x - l) + 1  # :12

    def add_tracer(self, tracer: ExpertTracer):
        self.tracer = tracer

    def predict(self, seq_id, expert_list, layer_idx) -> np.ndarray:  # :17-35
        self.tracer.update_entry(seq_id, expert_list, layer_idx)
        current_entry = self.tracer.get_entry(seq_id)
        expert_matrix = self.tracer.find_most_similar(current_entry.matrix, layer_idx)
        expert_matrix[:layer_idx, :] = 0
        for l in range(layer_idx, self.num_layers):
            expert_matrix[l] = (expert_matrix[l] + 1e-8) * self.layer_decay_func(l, layer_idx, self.num_layers)
        return expert_matrix


class ExpertPrefetcher:
    """memory/expert_prefetcher.py:12-59.  `archer_engine` is anything with `prefetch_hint(pairs, scores)` or the
    reference pair `replace_cache_candidates(ids)` / `enqueue_prefetch(id, gpu)` (then `expert_tensor_map` is used)."""

    def __init__(self, num_layers: int, num_experts: int, num_encoder_layers: int = 0):
        self.num_layers, self.num_experts, self.num_encoder_layers = num_layers, num_experts, num_encoder_layers
        self.expert_tensor_map: Optional[Dict[Tuple[int, int], int]] = None
        self.archer_engine = None

    def set_archer_engine(self, archer_engine):
        self.archer_engine = archer_engine

    def ordered_requests(self, layer_id: int, expert_matrix: np.ndarray) -> List[Tuple[Tuple[int, int], float]]:
        """(layer, expert) with score > 0 for layers >= layer_id, sorted by descending score (stable)  -- :43-54"""
        reqs = []
        for i in range(layer_id, self.num_layers):
            for j in range(self.num_experts):
                if expert_matrix[i, j] > 0:
                    reqs.append(((i, j), float(expert_matrix[i, j])))
        return sorted(reqs, key=lambda x: x[1], reverse=True)

    def prefetch_experts(self, layer_id: int, expert_matrix: np.ndarray):  # :42-59
        reqs = self.ordered_requests(layer_id, expert_matrix)
        if hasattr(self.archer_engine, "prefetch_hint"):
            self.archer_engine.prefetch_hint([p for p, _ in reqs], [s for _, s in reqs])
            return
        tensor_ids = [self.expert_tensor_map[p] for p, _ in reqs]
        assert len(np.unique(tensor_ids)) == len(tensor_ids)
        self.archer_engine.replace_cache_candidates(tensor_ids)
        for tid in tensor_ids:
            gpu_id = self.archer_engine.get_node_default_device([tid])
            self.archer_engine.enqueue_prefetch(tid, gpu_id)

    def prefetch_experts_list(self, layer_id: int, expert_list: Sequence[int]):  # :29-34
        for j in expert_list:
            self.archer_engine.enqueue_prefetch(layer_id, j)

    def fetch_experts_lock_cache(self, layer_id: int, expert_list: Sequence[int]):  # :36-40
        self.archer_engine.replace_cache_candidates([(layer_id, j) for j in expert_list])


# --------------------------------------------------------------------------------------------------------------
# P6: the paper's "sparsity-aware" cache priority (moe_infinity/memory/expert_priority_score.py:84-172).  The
# reference never instantiates ExpertCache (runtime/model_offload.py:83 is commented out), so this is a policy
# *specification*; it is restated here, vectorised, for users who want to feed the C-ABI scheduler with it
# (e.g. as `prefetch_hint` scores or to choose `replace_cache_candidates`).
# --------------------------------------------------------------------------------------------------------------
def priority_score_matrix(expert_freq: Dict[Tuple[int, int], float], decoder_matrix: np.ndarray, current_layer: int,
                          total_layer: int) -> np.ndarray:
    """score[l, e] = topo_decay(l | current_layer) * normalised activations of the running sequence * normalised
    visit frequency, each term + 1e-6 (expert_priority_score.py:93-172).  `expert_freq` maps (expert, layer) -> visits.
    Returns the [L, E] matrix (the reference converts entries > 0 into a list of ExpertCacheEntry)."""
    L_, E_ = decoder_matrix.shape
    ne = total_layer // 2                                        # :92 num_encoder_layers
    freq = np.zeros((L_, E_), dtype=np.float64)
    for (e, l), v in expert_freq.items():                        # :96-98
        freq[l, e] = v
    if freq[ne:].sum() == 0:                                     # :100-104
        freq[ne:] = 1
    if freq[:ne].sum() == 0:
        freq[:ne] = 1
    freq = freq / freq.sum() + 1e-6                              # :106
    i = np.arange(L_, dtype=np.float64)
    first = -1.0 / ne * i + 1 if ne else np.ones(L_)             # decay_from_first(x, L)  :8
    last = 1.0 / (ne + 1) * (i - ne)                             # decay_from_last(x - ne, L)  :9
    topo = np.empty(L_, dtype=np.float64)
    enc = i < ne
    if current_layer < ne:                                       # :115-126
        topo[enc] = np.where(i[enc] > current_layer, first[enc], 1.0)
        topo[~enc] = last[~enc]
    else:                                                        # :127-138
        topo[enc] = first[enc]
        topo[~enc] = np.where(i[~enc] > current_layer, last[~enc], 1.0)
    topo = np.repeat(topo[:, None], E_, axis=1)
    topo = topo / topo.sum() + 1e-6                              # :139
    dec = decoder_matrix.astype(np.float64).copy()               # :161-171
    if dec.sum() == 0:
        dec = np.ones_like(dec)
    rows = dec.sum(axis=1, keepdims=True)
    dec = np.where(rows == 0, 1.0, dec)
    dec = dec / dec.sum(axis=1, keepdims=True)
    dec = dec / dec.sum() + 1e-6
    return topo * dec * freq                                     # :172
