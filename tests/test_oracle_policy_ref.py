"""CPU: the cache-policy oracle and the host logic of csrc/api.cu against a trace RECORDED FROM THE REFERENCE'S OWN ENGINE.

tests/golden/policy_ref_trace.json was produced by tools/ref_engine_harness.py --mode policy: the reference's
compiled `prefetch_op.so` (core/parallel/expert_dispatcher.cpp GPUFetchFunc :191-307, Node::SetDevice) replayed a seeded
sequence of (layer, active experts) requests with an HBM budget of `slots` experts; for every dispatched expert the
harness stored the `hit` flag wait_expert() returned (:219,301) and the set of GPU-resident experts afterwards
(is_tensor_on_device).  "sequential" records dispatch one expert per set_expected_queue(1)/enqueue/wait, which makes the
reference deterministic (every earlier expert has been unlocked by OutputFunc before the next victim scan).
Here: oracle/policy_oracle.py (policy "reference") and the real api.cu (host emulation, tests/host/sim) must reproduce the
hit flags and the resident sets exactly, including the clear_expert_cache_counts() call in the middle of the trace."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "policy_ref_trace.json")
pytestmark = pytest.mark.skipif(not os.path.exists(GOLD), reason="golden trace of the reference engine not recorded yet")

from oracle.policy_oracle import CacheOracle  # noqa: E402


def _load():
    with open(GOLD) as f:
        return json.load(f)


def test_policy_oracle_reproduces_reference_engine_sequential_trace():
    g = _load()
    cfg = g["config"]
    orc = CacheOracle(cfg["layers"], cfg["experts"], cfg["slots"], policy="reference")
    cleared = set(g["clear_counts_at"])
    last_n = -1
    for rec in g["sequential"]:
        if rec["n"] != last_n and rec["n"] in cleared:
            orc.clear_counts()
        last_n = rec["n"]
        (e, hit), = orc.dispatch(rec["layer"], [rec["expert"]])
        assert (e, int(hit)) == (rec["expert"], rec["hit"]), rec
        res = sorted([i // orc.E, i % orc.E] for i in range(orc.L * orc.E) if orc.resident[i])
        assert res == rec["resident_after"], (rec["n"], rec["layer"], rec["expert"])
    assert sum(r["hit"] for r in g["sequential"]) == orc.stats["hits"]


def test_api_cu_host_logic_reproduces_reference_engine_sequential_trace():
    sys.path.insert(0, os.path.join(HERE, "host", "sim"))
    import build_sim
    from moe_infinity_b200 import _lib as L
    so = build_sim.build()
    if so is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    lib = C.CDLL(so)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    g = _load()
    cfg_ = g["config"]
    Ln, E, H, I = cfg_["layers"], cfg_["experts"], 128, 128
    cfg = L.Config()
    cfg.struct_size = C.sizeof(L.Config)
    cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = Ln, E, H, I, 1
    cfg.dtype, cfg.expert_type, cfg.router, cfg.max_tokens = L.DTYPE_BF16, L.EXPERT_MIXTRAL, L.ROUTER_MIXTRAL, 16
    cfg.gate_dtype, cfg.num_slots, cfg.routed_scaling_factor = L.DTYPE_BF16, cfg_["slots"], 1.0
    cfg.cache_policy = L.CACHE_REFERENCE
    h = C.c_void_p()
    assert lib.b2m_ctx_create(C.byref(cfg), C.byref(h)) == 0
    blobs = {}
    rng = np.random.default_rng(0)
    for l in range(Ln):
        for e in range(E):
            blobs[(l, e)] = rng.integers(0, 255, 3 * H * I * 2, dtype=np.uint8)
            assert lib.b2m_register_expert(h, l, e, blobs[(l, e)].ctypes.data, blobs[(l, e)].nbytes) == 0
    x = np.zeros((4, H), dtype=np.uint16)
    out = np.zeros((4, H), dtype=np.uint16)
    cleared = set(g["clear_counts_at"])
    last_n = -1
    for rec in g["sequential"]:
        if rec["n"] != last_n and rec["n"] in cleared:
            assert lib.b2m_clear_expert_cache_counts(h) == 0
        last_n = rec["n"]
        l, e = rec["layer"], rec["expert"]
        before = lib.b2m_is_resident(h, l, e)
        lg = np.full((4, E), -30.0, dtype=np.float32)
        lg[:, e] = 5.0                                        # top-1 router: exactly this expert is active
        rc = lib.b2m_moe_forward(h, l, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, 4, 0, out.ctypes.data, None)
        assert rc == 0, lib.b2m_last_error(h)
        assert before == rec["hit"], rec
        res = sorted([ll, ee] for ll in range(Ln) for ee in range(E) if lib.b2m_is_resident(h, ll, ee))
        assert res == rec["resident_after"], (rec["n"], l, e)
    lib.b2m_ctx_destroy(h)


def test_batch_protocol_hit_flags():
    """dispatch_local's all-at-once enqueue: which experts of the layer are still locked when a later miss of the same
    layer scans for a victim depends on the reference's thread timing.  The hit flags do not (they are taken at fetch
    time, in queue order, and a victim is never an expert whose own fetch is still queued... unless it was already
    processed and released) -- they must agree with the oracle wherever the two recorded repetitions of the reference
    agree with each other on the resident set."""
    g = _load()
    cfg = g["config"]
    orc = CacheOracle(cfg["layers"], cfg["experts"], cfg["slots"], policy="reference")
    # bring the oracle to the state the reference was in when the batch protocol started
    cleared = set(g["clear_counts_at"])
    last_n = -1
    for rec in g["sequential"]:
        if rec["n"] != last_n and rec["n"] in cleared:
            orc.clear_counts()
        last_n = rec["n"]
        orc.dispatch(rec["layer"], [rec["expert"]])
    agree, total = 0, 0
    for rec in g["batch"]:
        req = g["trace"][rec["n"]]
        got = orc.dispatch(rec["layer"], req["experts"])
        res = sorted([i // orc.E, i % orc.E] for i in range(orc.L * orc.E) if orc.resident[i])
        total += 1
        same = [int(h) for _, h in got] == rec["hits"] and res == rec["resident_after"]
        agree += int(same)
        if not same:
            # re-synchronise the oracle with what the reference actually did, so one timing-dependent eviction does not
            # cascade through the rest of the comparison
            want = {tuple(p) for p in rec["resident_after"]}
            for i in range(orc.L * orc.E):
                now = (i // orc.E, i % orc.E) in want
                if orc.resident[i] != now:
                    orc.resident[i] = now
            orc.free = orc.nslots - len(want)
    print(f"batch protocol: {agree}/{total} layer dispatches identical to the oracle's all-experts-locked semantics")
    assert agree >= 0.5 * total
