"""Generate tests/golden/reference_results.pt: what the reference's own code returns on the inputs of the tests that compare
against it, so that those comparisons run without the reference tree.

Run:  B2M_REFERENCE_ROOT=<reference checkout> python tests/golden/make_ref_golden.py
Needs the reference tree (for the literal Python policy classes, tests/shims/ref_loader.py) and
oracle/_ref/ref_expert_module.so (the reference's expert modules and index code compiled as-is, oracle/ref_build/Makefile).
Stored, per test:
  * predictor / prefetcher / priority score (moe_infinity/memory/*.py): the literal classes' outputs on the seeded inputs
    tests/test_memory_policy.py regenerates;
  * expert modules (core/parallel/expert_module.cpp): a SHA-256 of every output's bytes plus its dtype and shape -- the
    tests demand bit equality, so a digest is as strict as the tensor and a fraction of its size;
  * tensor index (core/aio/archer_tensor_index.cpp): the reference writer's file and the reference reader's entries for
    the seeded tensor sets of tests/test_store_format.py.
"""
from __future__ import annotations

import contextlib
import hashlib
import io
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
for p in (ROOT, os.path.join(ROOT, "moe-infinity_b200"), TESTS, os.path.join(TESTS, "shims"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(HERE, "reference_results.pt")

# inputs shared with the tests
PREDICTOR_SEEDS = (0, 1, 2)
PREDICTOR_SHAPE = dict(L=6, E=8, cap=12, n_lib=9, steps=3)
PREFETCH_SHAPE = dict(L=5, E=4, seed=3, layer=2)
PRIORITY_LAYERS = (0, 2, 3, 5)
PRIORITY_SHAPE = dict(L=6, E=4)
EXPERT_SHAPES = [(32, 48, 1), (64, 40, 13), (72, 136, 4), (256, 512, 33)]
STORE_SEEDS = range(4)
STORE_TENSORS = 25


def digest(t: torch.Tensor) -> dict:
    t = t.detach().contiguous()
    raw = t.reshape(-1).view(torch.uint8).numpy().tobytes() if t.numel() else b""
    return {"sha256": hashlib.sha256(raw).hexdigest(), "dtype": str(t.dtype), "shape": tuple(t.shape)}


def library(rng, n, L, E):
    lib = rng.integers(0, 6, size=(n, L, E)).astype(np.float32)
    lib[:, :, 0] += 1.0   # no all-zero rows
    return lib


def priority_inputs(current_layer):
    L, E = PRIORITY_SHAPE["L"], PRIORITY_SHAPE["E"]
    rng = np.random.default_rng(current_layer)
    dec = rng.integers(0, 4, size=(L, E)).astype(np.float64)
    dec[1] = 0                                           # an all-zero layer row
    freq = {(int(e), int(l)): float(rng.integers(0, 5)) for l in range(L) for e in range(E) if rng.random() < 0.6}
    return dec, freq


def prefetch_inputs():
    L, E = PREFETCH_SHAPE["L"], PREFETCH_SHAPE["E"]
    rng = np.random.default_rng(PREFETCH_SHAPE["seed"])
    matrix = rng.random((L, E)) * (rng.random((L, E)) > 0.3)
    tmap = {(l, e): 100 + l * E + e for l in range(L) for e in range(E)}
    return matrix, tmap


def expert_case(et, dt, H, I, n, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.1).to(dt)  # noqa: E731
    if et == 0:
        ws = [r(I, H), r(H, I)]
    elif et == 4:
        ws = [r(I, H), r(H, I), r(I, H)]
    elif et in (1, 5):
        ws = [r(I, H), r(I, H), r(H, I)]
    else:
        ws = [r(I, H), r(I), r(H, I), r(H)]
    return ws, torch.randn(n, H, generator=g).to(dt)


def random_tensors(seed, n):
    g = torch.Generator().manual_seed(seed)
    dts = [torch.bfloat16, torch.float16, torch.float32, torch.int64, torch.uint8, torch.bool, torch.float64]
    out = {}
    for i in range(n):
        dt = dts[int(torch.randint(0, len(dts), (1,), generator=g))]
        rank = int(torch.randint(0, 4, (1,), generator=g))
        shape = [int(torch.randint(1, 40, (1,), generator=g)) for _ in range(rank)]
        t = (torch.randn(shape, generator=g) * 10)
        t = (t > 0) if dt == torch.bool else t.to(dt)
        out[int(torch.randint(0, 2 ** 31, (1,), generator=g)) * 2 + (i % 2)] = t
    return out


class PrefetchRecorder:
    """The archer engine as the prefetcher sees it: records the candidates and the prefetch queue."""

    def __init__(self):
        self.cands, self.enq = None, []

    def replace_cache_candidates(self, ids):
        self.cands = list(ids)

    def get_node_default_device(self, ids):
        return 0

    def enqueue_prefetch(self, tid, gpu):
        self.enq.append(tid)


@contextlib.contextmanager
def _cpu_only_torch():
    """The literal ExpertTracer allocates on cuda:0 (expert_tracer.py:33-35,104); run it on CPU."""
    zeros, to = torch.zeros, torch.Tensor.to

    def zeros_cpu(*a, **k):
        k.pop("device", None)
        return zeros(*a, **k)

    def to_cpu(self, *a, **k):
        if any(isinstance(x, str) and x == "cpu" for x in a):
            return self.clone()
        a = tuple(x for x in a if not (isinstance(x, str) and x.startswith("cuda")))
        if not a and not k:
            return self
        return to(self, *a, **k)

    torch.zeros, torch.Tensor.to = zeros_cpu, to_cpu
    try:
        yield
    finally:
        torch.zeros, torch.Tensor.to = zeros, to


def _cfg(L, E):
    import types
    return types.SimpleNamespace(architectures=["MixtralForCausalLM"], num_hidden_layers=L, num_local_experts=E)


def policy_results(ns):
    import importlib
    res = {"predictor": {}, "priority": {}}
    L, E, cap, n_lib, steps = (PREDICTOR_SHAPE[k] for k in ("L", "E", "cap", "n_lib", "steps"))
    for seed in PREDICTOR_SEEDS:
        rng = np.random.default_rng(seed)
        lib = library(rng, n_lib, L, E)
        with _cpu_only_torch():
            ns.expert_tracer.ExpertTracer._instance = None
            rt = ns.expert_tracer.ExpertTracer(cap, _cfg(L, E))
            rt.trace_collection[:n_lib] = torch.from_numpy(lib)
            rp = ns.expert_predictor.ExpertPredictor(_cfg(L, E))
            rp.add_tracer(rt)
            rs = rt.create_entry()
            preds = []
            for _ in range(steps):
                for layer in range(L):
                    experts = rng.integers(0, E, size=(4, 2))
                    preds.append(np.asarray(rp.predict(rs, torch.from_numpy(experts), layer), dtype=np.float64))
            res["predictor"][seed] = {"predictions": np.stack(preds), "matrix": np.asarray(rt.get_entry(rs).matrix),
                                      "collection_access": np.asarray(rt.collection_access)}
    matrix, tmap = prefetch_inputs()
    with contextlib.redirect_stdout(io.StringIO()):
        rp = ns.expert_prefetcher.ExpertPrefetcher(_cfg(PREFETCH_SHAPE["L"], PREFETCH_SHAPE["E"]))
    rp.expert_tensor_map = tmap
    rec = PrefetchRecorder()
    rp.set_archer_engine(rec)
    rp.prefetch_experts(PREFETCH_SHAPE["layer"], matrix)
    res["prefetch"] = {"candidates": rec.cands, "enqueued": rec.enq}
    ps = importlib.import_module("moe_infinity.memory.expert_priority_score")
    ent = importlib.import_module("moe_infinity.memory.expert_entry")
    L, E = PRIORITY_SHAPE["L"], PRIORITY_SHAPE["E"]
    for cl in PRIORITY_LAYERS:
        dec, freq = priority_inputs(cl)
        entry = ent.ExpertTraceEntry("s", dec.copy(), 0, 0)
        m = np.zeros((L, E))
        for ce in ps.priority_score(freq, set(), set(), entry, cl, L):
            m[ce.layer_idx, ce.expert_idx] = ce.r
        res["priority"][cl] = m
    return res


def expert_results(R):
    import expert_cases as C
    torch.set_num_threads(1)
    res = {}
    for et in range(6):
        for di in range(3):
            dt = C.DT[di]
            for i, (H, I, n) in enumerate(EXPERT_SHAPES):
                ws, x = expert_case(et, dt, H, I, n, 1000 + 17 * et + 5 * di + i)
                res[(et, di, i)] = digest(R.expert_forward(et, di, ws, x))
    ws, x = expert_case(0, torch.float32, 64, 96, 6, 77)
    res["switch_cast"] = digest(R.expert_forward(0, 1, ws, x.to(torch.bfloat16)))
    return res


def store_results(R):
    from moe_infinity_b200.store import ArcherTensorStore
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for seed in STORE_SEEDS:
            tensors = random_tensors(seed, STORE_TENSORS)
            store = ArcherTensorStore(os.path.join(tmp, f"s{seed}"))
            for tid, t in tensors.items():
                store.store_tensor(tid, t, flush=False)
            store.flush()
            read = {e[0]: tuple(e[1:]) for e in R.index_deserialize(store.index_path)}
            ref_path = os.path.join(tmp, f"ref_index{seed}")
            R.index_serialize(ref_path, [(tid, store.index[tid].file_id, store.index[tid].offset, t) for tid, t in tensors.items()])
            with open(ref_path, "rb") as f:
                res[seed] = {"reader_entries": read, "writer_bytes": f.read()}
    return res


def main():
    import ref_loader
    from oracle import ref_module
    R = ref_module.load()
    assert R is not None, "oracle/_ref/ref_expert_module.so missing (oracle/ref_build/Makefile builds it)"
    assert ref_loader.available(), "reference tree not found (set B2M_REFERENCE_ROOT)"
    out = {"policy": policy_results(ref_loader.load()), "expert": expert_results(R), "store": store_results(R)}
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
