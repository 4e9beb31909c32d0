"""CPU: the HOST logic of the C-ABI layer (moe-infinity_b200/csrc/api.cu, compiled unchanged) executed without a GPU.

tests/host/sim/ links api.cu against a host emulation of the CUDA runtime (device memory = host memory, copies = memcpy,
streams/events complete immediately) and stand-in kernel launchers that compute the routing tables with plain loops and
RECORD every GEMM launch.  What is checked here is everything api.cu decides on the host:
  * the HBM expert cache reproduces oracle/policy_oracle.py's hit / miss / eviction sequence and residency map, with
    prefetch hints, protected candidates and wave splitting when one layer's active set exceeds the slot budget;
  * a staged slot really holds the expert's host blob (right bytes in the right slot after evictions and re-use);
  * launch planning: token-tile width, split-K / stream-K, programmatic-edge flags, slot tables handed to the kernels;
  * argument / state errors are reported through return codes + b2m_last_error, never by aborting.
The product library is not involved (it refuses to create a context without a GPU: tests/test_cabi_symbols.py)."""
from __future__ import annotations

import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from oracle.policy_oracle import CacheOracle  # noqa: E402

_SO = build_sim.build()
pytestmark = pytest.mark.skipif(_SO is None, reason="nvcc / g++ not available to build the host simulation")


@pytest.fixture(scope="module")
def sim():
    lib = C.CDLL(_SO)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.b2m_sim_take_log.restype, lib.b2m_sim_take_log.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t]
    lib.b2m_sim_h2d_bytes.restype = C.c_longlong
    lib.b2m_sim_live_allocs.restype = C.c_longlong
    return lib


class Ctx:
    """Minimal driver of the C ABI with host buffers (the simulation's 'device' pointers are host pointers)."""

    def __init__(self, lib, L_=3, E=8, H=128, I=256, k=2, max_tokens=64, expert_type=L.EXPERT_MIXTRAL, **kw):
        self.lib, self.L, self.E, self.H, self.I, self.k = lib, L_, E, H, I, k
        cfg = L.Config()
        cfg.struct_size = C.sizeof(L.Config)
        cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = L_, E, H, I, k
        cfg.dtype, cfg.expert_type, cfg.router, cfg.max_tokens = L.DTYPE_BF16, expert_type, kw.pop("router", L.ROUTER_MIXTRAL), max_tokens
        cfg.gate_dtype = L.DTYPE_BF16
        cfg.device_memory_ratio = 0.5
        cfg.routed_scaling_factor = 1.0
        for key, v in kw.items():
            setattr(cfg, key, v)
        self.h = C.c_void_p()
        self.rc = lib.b2m_ctx_create(C.byref(cfg), C.byref(self.h))
        self.blobs = {}

    def err(self):
        return (self.lib.b2m_last_error(self.h) or b"").decode()

    def close(self):
        if self.h:
            self.lib.b2m_ctx_destroy(self.h)
            self.h = C.c_void_p()

    def expert_bytes(self):
        return 3 * self.H * self.I * 2          # w1 | w2 | w3 (the Mixtral blob these tests register)

    def register_all(self, seed=0):
        rng = np.random.default_rng(seed)
        for l in range(self.L):
            for e in range(self.E):
                blob = rng.integers(0, 255, self.expert_bytes(), dtype=np.uint8)
                self.blobs[(l, e)] = blob
                assert self.lib.b2m_register_expert(self.h, l, e, blob.ctypes.data, blob.nbytes) == 0, self.err()

    def forward(self, layer, logits_f32):
        T = logits_f32.shape[0]
        x = np.zeros((T, self.H), dtype=np.uint16)
        out = np.zeros((T, self.H), dtype=np.uint16)
        lg = np.ascontiguousarray(logits_f32, dtype=np.float32)
        rc = self.lib.b2m_moe_forward(self.h, layer, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, out.ctypes.data, None)
        return rc

    def stats(self):
        s = L.Stats()
        assert self.lib.b2m_stats_get(self.h, C.byref(s)) == 0
        return s.as_dict()

    def counts(self):
        # straight from the workspace (host memory in the simulation); b2m_last_counts only answers after an offload-mode call
        p = C.c_void_p()
        assert self.lib.b2m_ws_ptr(self.h, L.WS["counts"], C.byref(p)) == 0, self.err()
        return list((C.c_int32 * self.E).from_address(p.value))

    def resident(self, l, e):
        return bool(self.lib.b2m_is_resident(self.h, l, e))

    def slot_bytes(self, l, e):
        p = C.c_void_p()
        assert self.lib.b2m_expert_dev_ptr(self.h, l, e, C.byref(p)) == 0
        return None if not p.value else np.ctypeslib.as_array((C.c_uint8 * self.expert_bytes()).from_address(p.value))


def take_log(lib):
    buf = C.create_string_buffer(1 << 20)
    lib.b2m_sim_take_log(buf, len(buf))
    return [ln for ln in buf.value.decode().split("\n") if ln]


def _kv(line):
    return {m.group(1): m.group(2) for m in re.finditer(r"(\w+)=(\[[^\]]*\]|\S+)", line)}


def test_cache_policy_matches_oracle_on_cpu(sim):
    for nslots, seed in ((10, 2), (9, 3), (8, 4)):
        c = Ctx(sim, num_slots=nslots)
        assert c.rc == 0, c.err()
        c.register_all(seed)
        orc = CacheOracle(c.L, c.E, nslots)
        rng = np.random.default_rng(seed)
        h2d0 = sim.b2m_sim_h2d_bytes()
        for step in range(12):
            for l in range(c.L):
                lg = rng.standard_normal((5, c.E)).astype(np.float32)
                before = {e: c.resident(l, e) for e in range(c.E)}
                assert c.forward(l, lg) == 0, c.err()
                cnt = c.counts()
                active = [e for e in range(c.E) if cnt[e] > 0]
                # the stand-in router is top-2 of the logits, lowest index on ties
                want = sorted(set(np.argsort(-lg, axis=1, kind="stable")[:, :2].flatten().tolist()))
                assert active == want
                assert [(e, before[e]) for e in active] == orc.dispatch(l, active), (nslots, step, l)
                for ll in range(c.L):
                    for e in range(c.E):
                        assert c.resident(ll, e) == orc.resident[ll * c.E + e]
                # every resident expert's slot holds exactly its host blob
                for e in active:
                    assert np.array_equal(c.slot_bytes(l, e), c.blobs[(l, e)])
        s = c.stats()
        for key in ("dispatches", "hits", "misses", "evictions"):
            assert s[key] == orc.stats[key], (nslots, key)
        assert s["h2d_bytes"] == s["misses"] * c.expert_bytes()
        assert s["host_syncs"] == 12 * c.L          # one count read-back per layer call (the reference's own sync point)
        lc = (C.c_int32 * c.E)()
        assert sim.b2m_last_counts(c.h, lc) == 0 and list(lc) == c.counts()
        assert s["resident"] <= nslots
        assert sim.b2m_sim_h2d_bytes() - h2d0 >= s["h2d_bytes"]
        c.close()


def _one_hot_logits(T, E, experts):
    lg = np.full((T, E), -30.0, dtype=np.float32)
    for t in range(T):
        lg[t, experts[t % len(experts)]] = 5.0
        lg[t, experts[(t + 1) % len(experts)]] = 4.0
    return lg


def test_reference_budget_charges_hits_on_cpu(sim):
    """expert_dispatcher.cpp:266 subtracts byte_size for every dispatched expert, hit or miss: with hits before the cache
    is full the budget runs out while physical slots are still free, and the next miss evicts (policy 'reference');
    B2M_CACHE_SLOTS evicts only when no slot is free."""
    for policy, name in ((L.CACHE_REFERENCE, "reference"), (L.CACHE_SLOTS, "slots")):
        c = Ctx(sim, L_=2, E=8, num_slots=6, cache_policy=policy)
        assert c.rc == 0, c.err()
        c.register_all(7)
        orc = CacheOracle(c.L, c.E, 6, policy=name)
        seq = [(0, [0, 1]), (0, [0, 1]), (0, [0, 1]), (1, [2, 3]), (1, [4, 5]), (0, [6, 7]), (1, [0, 1])]
        for l, ex in seq:
            before = {e: c.resident(l, e) for e in ex}
            assert c.forward(l, _one_hot_logits(4, c.E, ex)) == 0, c.err()
            assert [(e, before[e]) for e in ex] == orc.dispatch(l, ex)
            for ll in range(c.L):
                for e in range(c.E):
                    assert c.resident(ll, e) == orc.resident[ll * c.E + e], (name, l, ex, ll, e)
        s = c.stats()
        assert s["evictions"] == orc.stats["evictions"] and s["misses"] == orc.stats["misses"]
        if name == "reference":
            assert s["evictions"] > 0 and s["resident"] < 6     # budget used up by hits: evicts with free slots left
        c.close()


def test_activation_aware_policy_matches_oracle_on_cpu(sim):
    """B2M_CACHE_ACTIVATION_AWARE: victim = largest expected time to next use (layer distance + L*(1/f - 1)); api.cu and
    oracle/policy_oracle.py (policy 'activation_aware') agree on every hit flag and resident set of a seeded decode trace
    in which layers are visited in order."""
    for nslots, seed in ((10, 12), (13, 13)):
        c = Ctx(sim, L_=4, E=8, num_slots=nslots, cache_policy=L.CACHE_ACTIVATION_AWARE)
        assert c.rc == 0, c.err()
        c.register_all(seed)
        orc = CacheOracle(c.L, c.E, nslots, policy="activation_aware")
        rng = np.random.default_rng(seed)
        bias = rng.standard_normal((c.L, c.E)).astype(np.float32) * 1.5        # per-layer popular experts
        for step in range(14):
            for l in range(c.L):
                lg = rng.standard_normal((5, c.E)).astype(np.float32) + bias[l]
                before = {e: c.resident(l, e) for e in range(c.E)}
                assert c.forward(l, lg) == 0, c.err()
                cnt = c.counts()
                active = [e for e in range(c.E) if cnt[e] > 0]
                assert [(e, before[e]) for e in active] == orc.dispatch(l, active), (nslots, step, l)
                for ll in range(c.L):
                    for e in range(c.E):
                        assert c.resident(ll, e) == orc.resident[ll * c.E + e], (nslots, step, l, ll, e)
        s = c.stats()
        assert s["evictions"] == orc.stats["evictions"] > 0 and s["misses"] == orc.stats["misses"]
        c.close()


def test_lookahead_prefetch_stages_next_layers_experts_on_cpu(sim):
    """cfg.lookahead_prefetch: the routing call also applies the NEXT layer's router weight to this layer's input; the
    predicted experts come back with the counts (no extra synchronisation), are protected from eviction and staged on the
    prefetch stream; a correctly predicted expert is a hit (prefetch_useful) when its layer runs."""
    Ln, E, H = 3, 8, 128
    c = Ctx(sim, L_=Ln, E=E, H=H, num_slots=20, cache_policy=L.CACHE_ACTIVATION_AWARE, lookahead_prefetch=2,
            max_inflight_prefetch=16)
    assert c.rc == 0, c.err()
    c.register_all(3)
    rng = np.random.default_rng(3)
    # router weights (bf16) per layer: expert e of layer l likes direction e + l (so the prediction is checkable)
    gates = []
    for l in range(Ln):
        g = np.zeros((E, H), dtype=np.float32)
        for e in range(E):
            g[e, (e + l) % E] = 4.0
        gb = (g.view(np.uint32) >> 16).astype(np.uint16)            # exact in bf16
        gates.append(gb)
        assert sim.b2m_set_gate(c.h, l, gb.ctypes.data) == 0
    T = 4
    syncs0 = c.stats()["host_syncs"]
    for step in range(3):
        for l in range(Ln):
            xf = np.zeros((T, H), dtype=np.float32)
            for t in range(T):
                xf[t, (t + step) % E] = 3.0
                xf[t, (t + step + 3) % E] = 2.0
            x = (xf.view(np.uint32) >> 16).astype(np.uint16)
            out = np.zeros((T, H), dtype=np.uint16)
            take_log(sim)
            rc = sim.b2m_moe_forward(c.h, l, x.ctypes.data, None, 0, 0, T, 0, out.ctypes.data, None)
            assert rc == 0, c.err()
            look = (C.c_int32 * E)()
            assert sim.b2m_last_lookahead(c.h, look) == 0, c.err()
            nxt = (l + 1) % Ln
            want = np.zeros(E, dtype=int)
            for t in range(T):                                       # top-2 of the next layer's logits on this input
                lg = xf[t] @ (gates[nxt].astype(np.uint32) << 16).view(np.float32).T
                for e in np.argsort(-lg, kind="stable")[:2]:
                    want[e] += 1
            assert list(look) == want.tolist()
            assert sim.b2m_prefetch_drain(c.h) == 0
            for e in range(E):
                if want[e] > 0:
                    assert c.resident(nxt, e), (step, l, e)           # staged ahead of its layer
    s = c.stats()
    assert s["host_syncs"] - syncs0 == 3 * Ln                        # still one read-back per layer call
    assert s["prefetch_issued"] > 0 and s["prefetch_useful"] > 0
    assert s["prefetch_useful"] >= 0.8 * (s["prefetch_issued"] - 4)   # same inputs feed every layer here: predictions hold
    c.close()


def test_all_resident_mode_never_syncs_on_cpu(sim):
    c = Ctx(sim, num_slots=24)                 # L*E slots: every expert fits
    c.register_all(4)
    rng = np.random.default_rng(4)
    for step in range(3):
        for l in range(c.L):
            assert c.forward(l, rng.standard_normal((5, c.E)).astype(np.float32)) == 0, c.err()
    s = c.stats()
    assert s["host_syncs"] == 0 and s["evictions"] == 0 and s["resident"] == 24
    lc = (C.c_int32 * c.E)()
    assert sim.b2m_last_counts(c.h, lc) != 0 and "sync-free" in c.err()
    for (l, e), blob in c.blobs.items():
        assert np.array_equal(c.slot_bytes(l, e), blob)
    c.close()


def test_prefetch_hints_protect_and_count_on_cpu(sim):
    nslots = 11
    c = Ctx(sim, num_slots=nslots)
    c.register_all(9)
    orc = CacheOracle(c.L, c.E, nslots)
    rng = np.random.default_rng(0)
    for step in range(10):
        for l in range(c.L):
            lg = rng.standard_normal((4, c.E)).astype(np.float32)
            assert c.forward(l, lg) == 0, c.err()
            cnt = c.counts()
            orc.dispatch(l, [e for e in range(c.E) if cnt[e] > 0])
            nl = (l + 1) % c.L
            cand = rng.choice(c.E, size=3, replace=False).tolist()
            scores = rng.random(3).astype(np.float32)
            pairs = (C.c_int32 * 6)(*[v for e in cand for v in (nl, int(e))])
            assert sim.b2m_prefetch_hint(c.h, 3, pairs, scores.ctypes.data_as(C.POINTER(C.c_float))) == 0, c.err()
            assert sim.b2m_prefetch_drain(c.h) == 0, c.err()
            orc.prefetch_hint([(nl, int(e)) for e in cand], scores.tolist())
            for ll in range(c.L):
                for e in range(c.E):
                    assert c.resident(ll, e) == orc.resident[ll * c.E + e], (step, l, ll, e)
    s = c.stats()
    for key in ("dispatches", "hits", "misses", "evictions", "prefetch_issued", "prefetch_useful"):
        assert s[key] == orc.stats[key], key
    assert s["prefetch_issued"] > 0 and s["prefetch_useful"] > 0
    c.close()


def test_fewer_slots_than_active_experts_runs_in_waves_on_cpu(sim):
    """With fewer slots than activated experts the GEMMs are launched wave by wave, each against a slot row that names only
    that wave's experts (-1 elsewhere), and every activated expert is covered exactly once."""
    for nslots in (1, 2, 3):
        c = Ctx(sim, num_slots=nslots)
        c.register_all(13)
        orc = CacheOracle(c.L, c.E, nslots)
        rng = np.random.default_rng(nslots)
        take_log(sim)
        for step in range(3):
            for l in range(c.L):
                lg = rng.standard_normal((6, c.E)).astype(np.float32)
                assert c.forward(l, lg) == 0, c.err()
                cnt = c.counts()
                active = [e for e in range(c.E) if cnt[e] > 0]
                orc.dispatch(l, active)
                gemms = [_kv(ln) for ln in take_log(sim) if ln.startswith("gemm")]
                ups = [g for g in gemms if g["epi"] == "0"]
                assert len(ups) == len(gemms) // 2 and len(ups) >= -(-len(active) // nslots)
                covered = []
                for g in ups:
                    row = eval(g["slot_of"])
                    wave = [e for e in range(c.E) if row[e] >= 0]
                    assert 1 <= len(wave) <= nslots and len(set(row[e] for e in wave)) == len(wave)
                    covered += [e for e in wave if e in active]
                assert sorted(covered) == active          # each activated expert in exactly one wave
        s = c.stats()
        for key in ("dispatches", "hits", "misses", "evictions"):
            assert s[key] == orc.stats[key], (nslots, key)
        c.close()


def test_launch_planning_on_cpu(sim):
    """Token-tile width, split-K / stream-K and programmatic-edge flags chosen by api.cu (pick_nt / pick_ksplit)."""
    # Mixtral-8x7B shapes need 2.8 GB per layer of fake HBM; use the same ratios at 1/8 size: H=512, I=1792
    c = Ctx(sim, L_=1, E=8, H=512, I=1792, k=2, max_tokens=4096, num_slots=8)
    assert c.rc == 0, c.err()
    c.register_all(1)
    rng = np.random.default_rng(5)
    take_log(sim)
    plans = {}
    for T in (1, 8, 40, 300, 4096):
        assert c.forward(0, rng.standard_normal((T, c.E)).astype(np.float32)) == 0, c.err()
        lines = take_log(sim)
        route = _kv([ln for ln in lines if ln.startswith("route")][0])
        up, dn = [_kv(ln) for ln in lines if ln.startswith("gemm")]
        assert up["epi"] == "0" and dn["epi"] == "1" and up["dual"] == "1" and up["M"] == "1792" and dn["M"] == "512"
        assert eval(up["offsets"])[-1] == T * 2
        plans[T] = (int(up["nt"]), int(dn["nt"]), int(dn["ksplit"]), int(dn["stream_k"]), int(up["early_a"]), int(dn["early_a"]),
                    int(route["offsets_early"]), int(dn["dual_m"]))
    # decode-sized batches: 16-token tiles, split-K with the stream-K partition, both GEMMs on programmatic edges
    for T in (1, 8):
        nt, ntd, ks, sk, ea_up, ea_dn, early, dual_m = plans[T]
        assert nt == 16 and ntd == 16 and ks > 1 and sk == 1 and ea_up == 1 and ea_dn == 1 and early == 1 and dual_m == 0
    assert plans[300][0] in (64, 128) and plans[300][6] == 0
    # few weight-row tiles (H=512 -> 4 m-tiles): even at T=4096 the planner splits K to fill the SMs
    # 128-token tiles for the gate/up GEMM, 256 for the down GEMM
    assert plans[4096][0] == 128 and plans[4096][1] == 256 and plans[4096][2] > 1 and plans[4096][5] == 0 and plans[4096][6] == 0
    c.close()
    # prefill with Mixtral's hidden size (32 m-tiles x 8 experts x 4 token tiles = 1024 tiles): 256-token tiles once the
    # average expert sees >= 256 tokens in the down projection (unpaired: a 256-token tile already shares each weight tile
    # between 256 tokens), no split-K, no programmatic edges; the gate/up GEMM keeps 128-token tiles in both numerics modes
    # (its gate and up accumulators of a 256-token tile would not fit in a warpgroup's registers)
    for numerics, up_nt in ((L.NUMERICS_FP32, "128"), (L.NUMERICS_REFERENCE, "128")):
        c = Ctx(sim, L_=1, E=8, H=4096, I=256, k=2, max_tokens=4096, num_slots=8, numerics=numerics)
        assert c.rc == 0, c.err()
        c.register_all(2)
        take_log(sim)
        assert c.forward(0, rng.standard_normal((4096, c.E)).astype(np.float32)) == 0, c.err()
        up, dn = [_kv(ln) for ln in take_log(sim) if ln.startswith("gemm")]
        assert (up["nt"], dn["nt"], dn["ksplit"], dn["stream_k"], up["early_a"], dn["early_a"], dn["dual_m"]) == \
            (up_nt, "256", "1", "0", "0", "0", "0")
        c.close()


def test_bias_experts_plan_whole_k_on_cpu(sim):
    c = Ctx(sim, L_=1, E=4, H=128, I=256, k=2, num_slots=4, expert_type=L.EXPERT_NLLB)
    assert c.rc == 0, c.err()
    nbytes = 2 * 128 * 256 * 2 + (256 + 128) * 2
    blob = np.zeros(nbytes, dtype=np.uint8)
    assert sim.b2m_register_expert(c.h, 0, 0, blob.ctypes.data, nbytes - 2) != 0 and "bytes" in c.err()
    for e in range(4):
        assert sim.b2m_register_expert(c.h, 0, e, blob.ctypes.data, nbytes) == 0, c.err()
    take_log(sim)
    assert c.forward(0, np.random.default_rng(0).standard_normal((3, 4)).astype(np.float32)) == 0, c.err()
    up, dn = [_kv(ln) for ln in take_log(sim) if ln.startswith("gemm")]
    assert up["bias"] == "1" and dn["bias"] == "1" and dn["ksplit"] == "1" and dn["stream_k"] == "0" and up["dual"] == "0"
    c.close()


def test_errors_are_reported_not_fatal_on_cpu(sim):
    bad = Ctx(sim, top_k=9)
    assert bad.rc == L.B2M_EINVAL
    assert Ctx(sim, dtype=L.DTYPE_FP8).rc == L.B2M_EUNSUPPORTED
    assert Ctx(sim, expert_type=6).rc != 0
    c = Ctx(sim, num_slots=4)
    assert c.rc == 0
    lg = np.zeros((3, c.E), dtype=np.float32)
    assert c.forward(0, lg) != 0 and "registered" in c.err()            # experts never registered
    c.register_all(0)
    assert c.forward(7, lg) != 0                                           # layer out of range
    assert c.forward(0, np.zeros((65, c.E), dtype=np.float32)) != 0 and "capacity" in c.err()
    assert sim.b2m_run_experts(c.h, 0, 5, None) != 0 and "routing call" in c.err()
    assert c.forward(0, lg) == 0, c.err()                                  # the context is still usable
    assert sim.b2m_register_expert(c.h, 0, 0, c.blobs[(0, 0)].ctypes.data, 10) != 0
    c.close()
    assert sim.b2m_ctx_destroy(None) in (0, L.B2M_EINVAL)


def test_dirty_slot_row_refuses_stream_capture_on_cpu(sim):
    """A changed expert->slot row is uploaded from a reused pinned staging ring; captured into a graph that copy would replay
    stale bytes.  The library refuses instead (the decode graph is captured after one eager step)."""
    c = Ctx(sim, num_slots=4)
    c.register_all(0)
    lg = np.zeros((3, c.E), dtype=np.float32)
    sim.fake_set_capturing(1)
    try:
        assert c.forward(0, lg) == L.B2M_ESTATE and "capturing" in c.err()
    finally:
        sim.fake_set_capturing(0)
    assert c.forward(0, lg) == 0, c.err()
    c.close()


def test_disk_backed_experts_stream_through_the_staging_ring_on_cpu(sim, tmp_path, monkeypatch):
    """SURVEY §8f N3: experts registered on a reference-format store are staged disk -> pinned chunk ring -> slot on a miss
    (api.cu: copy_from_store over csrc/store_reader.cpp, both compiled as they are), mixed with host-backed experts; the
    right bytes land in the right slots through evictions, and a read error is a return code, not an abort."""
    import torch
    from moe_infinity_b200.store import ArcherTensorStore
    monkeypatch.setenv("B2M_DISK_CHUNK_BYTES", str(10 * 4096))          # 196608-byte blobs -> 5 chunks that cross tensor ends
    c = Ctx(sim, L_=2, num_slots=3)
    assert c.rc == 0
    st = ArcherTensorStore(str(tmp_path))
    rng = np.random.default_rng(5)
    ids_of, want = {}, {}
    tid = 100
    for l in range(c.L):
        for e in range(c.E):
            parts = [rng.integers(0, 255, c.H * c.I * 2, dtype=np.uint8) for _ in range(3)]      # w1 | w2 | w3
            want[(l, e)] = np.concatenate(parts)
            if e % 2 == 0:                                                 # even experts live on the store ...
                ids_of[(l, e)] = list(range(tid, tid + 3))
                for p_ in parts:
                    st.store_tensor(tid, torch.from_numpy(p_), flush=False)
                    tid += 1
    st.flush()
    store = C.c_void_p()
    assert sim.b2m_store_open(str(tmp_path).encode(), 3, 8192, 0, C.byref(store)) == 0
    for (l, e), blob in want.items():
        if (l, e) in ids_of:
            arr = (C.c_uint32 * 3)(*ids_of[(l, e)])
            assert sim.b2m_register_expert_on_store(c.h, l, e, store, arr, 3) == 0, c.err()
        else:                                                              # ... odd ones in host memory
            c.blobs[(l, e)] = blob
            assert sim.b2m_register_expert(c.h, l, e, blob.ctypes.data, blob.nbytes) == 0, c.err()
    bad = (C.c_uint32 * 2)(100, 101)
    assert sim.b2m_register_expert_on_store(c.h, 0, 0, store, bad, 2) == L.B2M_EINVAL and "bytes on the store" in c.err()
    bad = (C.c_uint32 * 1)(7)
    assert sim.b2m_register_expert_on_store(c.h, 0, 0, store, bad, 1) == L.B2M_EINVAL and "not in the index" in c.err()

    def route_to(experts):
        lg = np.full((len(experts), c.E), -30.0, dtype=np.float32)
        for t_, (a, b) in enumerate(experts):
            lg[t_, a], lg[t_, b] = 5.0, 4.0
        return lg

    seen = 0
    for step, (layer, pairs) in enumerate([(0, [(0, 1)]), (0, [(2, 3)]), (1, [(4, 6)]), (0, [(0, 2)]), (1, [(1, 4)]), (0, [(6, 7)])]):
        assert c.forward(layer, route_to(pairs)) == 0, c.err()
        for a in {x for p_ in pairs for x in p_}:
            assert c.resident(layer, a)
            assert np.array_equal(c.slot_bytes(layer, a), want[(layer, a)]), (step, layer, a)
            seen += 1
    s = c.stats()
    assert s["evictions"] > 0 and s["misses"] >= 9
    out4 = (C.c_uint64 * 4)()
    assert sim.b2m_store_stats(store, out4) == 0
    assert out4[0] > 0 and out4[0] % want[(0, 0)].nbytes == 0            # whole blobs came from the disk, in 5-chunk requests
    assert out4[3] == 5 * (out4[0] // want[(0, 0)].nbytes)
    # a store file that lost its tail: the miss fails with B2M_EIO, the expert is not marked resident, the context lives on
    with open(tmp_path / "archer_param_0", "r+b") as f:
        f.truncate(4096)
    victim = next(e for e in (0, 2, 4, 6) if not c.resident(1, e))
    other = next(e for e in (1, 3, 5, 7) if e != victim)
    for _ in range(5):                                                     # (more failures than slots: none may leak)
        assert c.forward(1, route_to([(victim, other)])) == L.B2M_EIO and "disk tier" in c.err()
        assert not c.resident(1, victim)
    assert c.forward(0, route_to([(1, 3)])) == 0, c.err()                  # host-backed experts still work
    assert np.array_equal(c.slot_bytes(0, 1), want[(0, 1)])
    c.close()
    assert sim.b2m_store_close(store) == 0


def test_fp32_experts_take_the_cuda_core_path_on_cpu(sim):
    """dtype int 1 (expert_module.h:21): 4-byte blobs, CUDA-core fp32 GEMMs with whole-K tiles, fp32 combine; the fused
    gate is refused (router logits come in), a mask row with more than top_k experts raises the sticky error."""
    c = Ctx(sim, L_=1, E=4, H=128, I=256, k=2, num_slots=4, dtype=L.DTYPE_F32, expert_type=L.EXPERT_SWITCH_GATED)
    assert c.rc == 0, c.err()
    rng = np.random.default_rng(3)
    nbytes = 3 * 128 * 256 * 4
    for e in range(4):
        blob = rng.integers(0, 255, nbytes, dtype=np.uint8)
        c.blobs[(0, e)] = blob
        assert sim.b2m_register_expert(c.h, 0, e, blob.ctypes.data, blob.nbytes) == 0, c.err()
    assert sim.b2m_register_expert(c.h, 0, 0, c.blobs[(0, 0)].ctypes.data, nbytes // 2) != 0     # 2-byte-sized blob refused
    take_log(sim)
    T = 6
    x = np.zeros((T, 128), dtype=np.float32)
    out = np.zeros((T, 128), dtype=np.float32)
    lg = rng.standard_normal((T, 4)).astype(np.float32)
    assert sim.b2m_moe_forward(c.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, out.ctypes.data, None) == 0, c.err()
    lines = take_log(sim)
    up, dn = [_kv(ln) for ln in lines if ln.startswith("gemm")]
    assert up["impl"] == "f32" and dn["impl"] == "f32" and up["dual"] == "1" and dn["ksplit"] == "1" and dn["stream_k"] == "0"
    assert any(ln.startswith("combine") and "dtype=1" in ln for ln in lines)   # launch_combine routes dtype 1 to the fp32 kernel
    assert sim.b2m_moe_forward(c.h, 0, x.ctypes.data, None, 0, 0, T, 0, out.ctypes.data, None) == L.B2M_EUNSUPPORTED
    # a mask naming 3 experts for a token of a top-2 context is reported, not truncated silently
    mask = np.zeros((T, 4), dtype=np.uint8)
    mask[:, :2] = 1
    mask[3, 2] = 1
    assert sim.b2m_route_from_mask(c.h, 0, x.ctypes.data, mask.ctypes.data, T, None) == 0, c.err()
    assert sim.b2m_check_errors(c.h, None) == L.B2M_EINVAL and "top_k" in c.err()
    assert sim.b2m_check_errors(c.h, None) == 0          # sticky word cleared by the report
    c.close()


def test_context_releases_everything_on_cpu(sim):
    live0 = sim.b2m_sim_live_allocs()
    for _ in range(3):
        c = Ctx(sim, num_slots=6, shared_inter=0)
        c.register_all(2)
        assert c.forward(1, np.random.default_rng(1).standard_normal((9, c.E)).astype(np.float32)) == 0
        c.close()
    assert sim.b2m_sim_live_allocs() == live0, "device / pinned allocations leaked across ctx_create/destroy"


def test_chunked_copies_and_pinned_experts_on_cpu(sim):
    """h2d_chunk_bytes splits a staging copy into many pieces (so a miss can overtake a prefetch between pieces): the slot
    must still end up holding the whole blob.  Experts pinned with b2m_make_resident(flags=1) are never chosen as victims."""
    c = Ctx(sim, num_slots=9, h2d_chunk_bytes=64 * 1024)
    c.register_all(21)
    for e in (0, 1):
        assert sim.b2m_make_resident(c.h, 0, e, 1, None) == 0, c.err()       # pin (0,0) and (0,1)
    rng = np.random.default_rng(21)
    for step in range(12):
        for l in range(c.L):
            lg = rng.standard_normal((6, c.E)).astype(np.float32)
            lg[:, :2] -= 10.0                                                  # the pinned experts are never routed to
            assert c.forward(l, lg) == 0, c.err()
            cnt = c.counts()
            for e in range(c.E):
                if cnt[e] > 0:
                    assert np.array_equal(c.slot_bytes(l, e), c.blobs[(l, e)])
            assert c.resident(0, 0) and c.resident(0, 1), "a pinned expert was evicted"
    s = c.stats()
    assert s["evictions"] > 10 and s["h2d_bytes"] == (s["misses"] + 2) * c.expert_bytes()   # + the two explicit stagings
    for e in (0, 1):
        assert np.array_equal(c.slot_bytes(0, e), c.blobs[(0, e)])
    c.close()


def test_reference_prefetch_pair_and_count_reset_on_cpu(sim):
    """replace_cache_candidates + enqueue_prefetch (archer_prefetch_handle.cpp:195-218) and clear_expert_cache_counts
    (interface_example.py:39) against the policy oracle."""
    nslots = 10
    c = Ctx(sim, num_slots=nslots)
    c.register_all(33)
    orc = CacheOracle(c.L, c.E, nslots)
    rng = np.random.default_rng(33)
    for step in range(9):
        for l in range(c.L):
            lg = rng.standard_normal((4, c.E)).astype(np.float32)
            assert c.forward(l, lg) == 0, c.err()
            cnt = c.counts()
            orc.dispatch(l, [e for e in range(c.E) if cnt[e] > 0])
            nl = (l + 1) % c.L
            cand = [(nl, int(e)) for e in rng.choice(c.E, size=2, replace=False)]
            flat = (C.c_int32 * 4)(*[v for pr in cand for v in pr])
            assert sim.b2m_replace_cache_candidates(c.h, 2, flat) == 0, c.err()
            orc.replace_cache_candidates(cand)
            for (ll, e) in cand:
                assert sim.b2m_enqueue_prefetch(c.h, ll, e) == 0, c.err()
            assert sim.b2m_prefetch_drain(c.h) == 0, c.err()
            orc.prefetch(cand)
            for ll in range(c.L):
                for e in range(c.E):
                    assert c.resident(ll, e) == orc.resident[ll * c.E + e], (step, l, ll, e)
        if step == 4:
            assert sim.b2m_clear_expert_cache_counts(c.h) == 0
            orc.clear_counts()
    s = c.stats()
    for key in ("dispatches", "hits", "misses", "evictions", "prefetch_issued", "prefetch_useful"):
        assert s[key] == orc.stats[key], key
    c.close()


def test_staged_calls_and_deepseek_shared_experts_on_cpu(sim):
    """The reference-compatible staged sequence (set_inputs -> enqueue/wait -> python combine = b2m_route_from_mask ->
    b2m_run_experts -> b2m_expert_outputs) and the DeepSeek flow with shared experts forked beside the routed path."""
    E, H, I, T = 8, 128, 128, 7
    c = Ctx(sim, L_=2, E=E, H=H, I=I, k=3, num_slots=16, expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY,
            shared_inter=2 * I, gate_dtype=L.DTYPE_F32)
    assert c.rc == 0, c.err()
    c.register_all(5)
    shared = np.zeros(3 * H * 2 * I * 2, dtype=np.uint8)
    assert sim.b2m_register_shared(c.h, 0, shared.ctypes.data, shared.nbytes - 16) != 0
    for l in range(2):
        assert sim.b2m_register_shared(c.h, l, shared.ctypes.data, shared.nbytes) == 0, c.err()
    take_log(sim)
    scores = np.random.default_rng(1).random((T, E)).astype(np.float32)
    x = np.zeros((T, H), dtype=np.uint16)
    out = np.zeros((T, H), dtype=np.uint16)
    assert sim.b2m_moe_forward(c.h, 1, x.ctypes.data, scores.ctypes.data, 2, L.DTYPE_F32, T, 0, out.ctypes.data, None) == 0, c.err()
    lines = take_log(sim)
    gemms = [_kv(ln) for ln in lines if ln.startswith("gemm")]
    assert len(gemms) == 4
    shared_g = [g for g in gemms if g["single_n"] == str(T)]
    assert len(shared_g) == 2 and all(g["single_slot"] == "1" for g in shared_g) and shared_g[0]["M"] == str(2 * I)
    assert [ln for ln in lines if ln.startswith("combine")] == [f"combine T={T} mode=1 shared=1 ep_collect=0 dtype=0"]
    # bf16 scores are refused (modeling_deepseek.py:473 computes them in fp32)
    assert sim.b2m_moe_forward(c.h, 1, x.ctypes.data, scores.ctypes.data, 2, L.DTYPE_BF16, T, 0, out.ctypes.data, None) != 0
    assert "fp32" in c.err()
    take_log(sim)
    # staged calls from a dense mask
    mask = np.zeros((T, E), dtype=np.uint8)
    mask[:, 2] = 1
    mask[::2, 5] = 1
    assert sim.b2m_route_from_mask(c.h, 0, x.ctypes.data, mask.ctypes.data, T, None) == 0, c.err()
    assert sim.b2m_run_experts_ex(c.h, 0, T, 1, None) == 0, c.err()            # gate/up phase only
    assert sim.b2m_run_experts_ex(c.h, 0, T, 2, None) == 0, c.err()            # down phase
    rows = np.zeros((T * 3, H), dtype=np.uint16)
    offs = (C.c_int * (E + 1))()
    assert sim.b2m_expert_outputs(c.h, T, rows.ctypes.data, offs, None) == 0, c.err()
    assert list(offs) == [0, 0, 0, T, T, T, T + 4, T + 4, T + 4]
    lines = take_log(sim)
    assert [ln.split()[0] for ln in lines] == ["route_from_mask", "gemm", "gemm", "cast_rows"]
    assert _kv(lines[1])["epi"] == "0" and _kv(lines[2])["epi"] == "1" and _kv(lines[1])["early_a"] == "0"
    c.close()


def test_expert_parallel_call_sequence_and_errors_on_cpu(sim):
    """Host side of the NCCL-style expert-parallel sequence (include/b2m.h: route -> ep_pack -> exchange -> ep_regroup ->
    run_experts -> ep_ungroup -> exchange -> ep_unpack -> combine): argument checks, the switch to EP mode (local experts
    all resident, never the on-demand path, no count read-back) and the peer-to-peer set-up failing cleanly when CUDA IPC
    is unavailable (the emulated runtime reports cudaErrorNotSupported; ep.py then falls back to NCCL)."""
    nranks, rank, T = 2, 1, 6
    E, H, k = 8, 128, 2
    c = Ctx(sim, L_=1, E=E, H=H, I=128, k=k, num_slots=4, max_tokens=64)       # this rank owns experts 4..7
    assert c.rc == 0, c.err()
    rng = np.random.default_rng(3)
    for e in range(4, 8):
        blob = rng.integers(0, 255, c.expert_bytes(), dtype=np.uint8)
        c.blobs[(0, e)] = blob
        assert sim.b2m_register_expert(c.h, 0, e, blob.ctypes.data, blob.nbytes) == 0, c.err()
        assert sim.b2m_make_resident(c.h, 0, e, 1, None) == 0, c.err()
    cap = T * k
    rows = np.zeros((nranks, cap + 1, H), dtype=np.uint16)
    x = np.zeros((T, H), dtype=np.uint16)
    lg = rng.standard_normal((T, E)).astype(np.float32)
    assert sim.b2m_route(c.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == 0, c.err()
    assert sim.b2m_ep_pack(c.h, nranks, rank, cap - 1, T, rows.ctypes.data, None, None) != 0 and "cap" in c.err()
    assert sim.b2m_ep_pack(c.h, 3, rank, cap, T, rows.ctypes.data, None, None) != 0             # 8 experts over 3 ranks
    assert sim.b2m_ep_pack(c.h, nranks, 2, cap, T, rows.ctypes.data, None, None) != 0           # rank out of range
    take_log(sim)
    assert sim.b2m_ep_pack(c.h, nranks, rank, cap, T, rows.ctypes.data, None, None) == 0, c.err()
    assert sim.b2m_ep_regroup(c.h, nranks, rank, cap, nranks * T, rows.ctypes.data, None, None) == 0, c.err()
    syncs0 = c.stats()["host_syncs"]
    assert sim.b2m_run_experts(c.h, 0, nranks * T, None) == 0, c.err()
    assert sim.b2m_ep_ungroup(c.h, nranks, rank, cap, rows.ctypes.data, None) == 0, c.err()
    assert sim.b2m_ep_unpack(c.h, nranks, rank, cap, T, rows.ctypes.data, None) == 0, c.err()
    out = np.zeros((T, H), dtype=np.uint16)
    assert sim.b2m_combine(c.h, 0, x.ctypes.data, T, out.ctypes.data, None) == 0, c.err()
    names = [ln.split()[0] for ln in take_log(sim)]
    assert names == ["ep_pack", "ep_regroup", "gemm", "gemm", "ep_ungroup", "ep_unpack", "combine"]
    s = c.stats()
    assert s["host_syncs"] == syncs0 and s["misses"] == 0 and s["evictions"] == 0      # EP mode: never the on-demand path
    # an unregistered local expert is an error in EP mode, not a silent skip
    c2 = Ctx(sim, L_=1, E=E, H=H, I=128, k=k, num_slots=8, max_tokens=64)
    handle = (C.c_char * 64)()
    assert sim.b2m_ep_p2p_init(c2.h, nranks, rank, cap, handle) != 0 and c2.err() != ""
    assert sim.b2m_route(c2.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == 0   # context still usable
    c.close()
    c2.close()


def test_expert_parallel_direct_layer_on_cpu(sim):
    """b2m_ep_p2p_layer, host side, two ranks in one process (the emulated CUDA IPC hands out plain pointers): the layer is
    four launches -- one routing call (gate/top-k that also claims rows in the owners' per-expert regions and stores them),
    a gate/up GEMM that waits for the peers, reads the row counters and clears the accumulator, a down GEMM that signals and
    resets the counters, a combine that reads the owners' outputs in place."""
    sim.b2m_sim_enable_ipc(1)
    try:
        nranks, T, E, H, I, k = 2, 6, 8, 128, 128, 2
        cap = T * k
        ctxs, handles = [], []
        rng = np.random.default_rng(9)
        for rank in range(nranks):
            c = Ctx(sim, L_=1, E=E, H=H, I=I, k=k, num_slots=E // nranks, max_tokens=nranks * T)
            assert c.rc == 0, c.err()
            for e in range(rank * E // nranks, (rank + 1) * E // nranks):
                blob = rng.integers(0, 255, c.expert_bytes(), dtype=np.uint8)
                c.blobs[(0, e)] = blob
                assert sim.b2m_register_expert(c.h, 0, e, blob.ctypes.data, blob.nbytes) == 0, c.err()
                assert sim.b2m_make_resident(c.h, 0, e, 1, None) == 0, c.err()
            h = (C.c_char * 64)()
            assert sim.b2m_ep_p2p_init(c.h, nranks, rank, cap, h) == 0, c.err()
            ctxs.append(c)
            handles.append(h)
        for c in ctxs:
            for peer in range(nranks):
                assert sim.b2m_ep_p2p_open(c.h, peer, handles[peer]) == 0, c.err()
        x = np.zeros((T, H), dtype=np.uint16)
        out = np.zeros((T, H), dtype=np.uint16)
        lg = rng.standard_normal((T, E)).astype(np.float32)
        for rank, c in enumerate(ctxs):
            take_log(sim)
            assert sim.b2m_ep_p2p_layer(c.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, out.ctypes.data, None) == 0, c.err()
            lines = take_log(sim)
            assert [ln.split()[0] for ln in lines] == ["route", "gemm", "gemm", "combine"]
            assert _kv(lines[0])["ep_dispatch"] == "1" and _kv(lines[0])["ep_direct"] == "1"
            up, dn = _kv(lines[1]), _kv(lines[2])
            R = nranks * cap                                       # rows of one expert region (its worst case)
            assert up["ep_rows"] == dn["ep_rows"] == str(R) and up["ep_first"] == str(rank * 4) and up["ep_el"] == "4"
            assert (up["ep_wait"], up["ep_signal"], dn["ep_wait"], dn["ep_signal"]) == ("1", "0", "0", "1")
            assert up["ep_cnt"] == dn["ep_cnt"] == "1"
            assert up["nt"] == dn["nt"] == "16" and up["dual"] == "1" and dn["epi"] == "1"    # ~2*T_total*k/E = 6 rows per expert expected
            assert up["grid"] == "4" and dn["grid"] == "132"      # 4 experts x 1 weight-row tile: the gate/up grid is sized to the expected tile list
            assert (dn["ksplit"] == "1") == (up["ep_zero"] == "0")          # the accumulator is cleared iff the down GEMM splits K
            assert "ep_direct=1" in lines[3] and _kv(lines[3])["ep_collect"] == "1"
            assert sim.b2m_ep_p2p_layer(c.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T + 1, out.ctypes.data, None) != 0
        for c in ctxs:
            c.close()
        # DeepSeek shared experts are outside the direct mode -> the seven-launch sequence (six here: route is one call)
        c = Ctx(sim, L_=1, E=64, H=H, I=I, k=k, num_slots=32, max_tokens=nranks * T, expert_type=L.EXPERT_DEEPSEEK,
                router=L.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I, gate_dtype=L.DTYPE_F32)
        assert c.rc == 0, c.err()
        for e in range(32):
            blob = rng.integers(0, 255, c.expert_bytes(), dtype=np.uint8)
            c.blobs[(0, e)] = blob
            assert sim.b2m_register_expert(c.h, 0, e, blob.ctypes.data, blob.nbytes) == 0, c.err()
            assert sim.b2m_make_resident(c.h, 0, e, 1, None) == 0, c.err()
        shared = np.zeros(3 * H * 2 * I * 2, dtype=np.uint8)
        assert sim.b2m_register_shared(c.h, 0, shared.ctypes.data, shared.nbytes) == 0, c.err()
        h = (C.c_char * 64)()
        assert sim.b2m_ep_p2p_init(c.h, nranks, 0, cap, h) == 0, c.err()
        assert sim.b2m_ep_p2p_open(c.h, 1, h) == 0, c.err()                 # loop-back "peer": enough for the call sequence
        sc64 = rng.random((T, 64)).astype(np.float32)
        take_log(sim)
        assert sim.b2m_ep_p2p_layer(c.h, 0, x.ctypes.data, sc64.ctypes.data, 2, L.DTYPE_F32, T, out.ctypes.data, None) == 0, c.err()
        names = [ln.split()[0] for ln in take_log(sim)]
        assert names[:2] == ["route", "ep_regroup"] and "ep_ungroup" in names and names[-1] == "combine"
        c.close()
    finally:
        sim.b2m_sim_enable_ipc(0)


def test_device_tracer_call_wiring_on_cpu(sim):
    """b2m_trace_*: argument / state checks, one predictor launch per call, and -- in offload mode with auto_prefetch --
    the hint matrix riding back with the next per-layer count read-back into the prefetch scheduler (no extra sync)."""
    c = Ctx(sim, L_=3, E=8, num_slots=10)
    assert c.rc == 0, c.err()
    c.register_all(1)
    assert sim.b2m_trace_update_predict(c.h, 0, 0, 1, 1, None) == L.B2M_ESTATE            # not initialised
    assert sim.b2m_trace_init(c.h, 16, 4, 1) == 0, c.err()
    assert sim.b2m_trace_init(c.h, 16, 4, 1) == L.B2M_ESTATE
    lib = np.ones((2, 3, 8), dtype=np.float32)
    assert sim.b2m_trace_load(c.h, 17, lib.ctypes.data) != 0
    assert sim.b2m_trace_load(c.h, 2, lib.ctypes.data) == 0, c.err()
    back = np.zeros((3, 8), dtype=np.float32)
    assert sim.b2m_trace_read(c.h, 3, 1, back.ctypes.data) == 0 and back.sum() == 24
    assert sim.b2m_trace_reset_seq(c.h, 4, None) != 0 and sim.b2m_trace_reset_seq(c.h, 3, None) == 0
    T = 4
    lg = np.random.default_rng(0).standard_normal((T, 8)).astype(np.float32)
    x = np.zeros((T, c.H), dtype=np.uint16)
    assert sim.b2m_route(c.h, 1, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == 0, c.err()
    assert sim.b2m_trace_update_predict(c.h, 1, 0, 3, 1, None) == L.B2M_ESTATE            # 3 x 1 tokens != T
    assert sim.b2m_trace_update_predict(c.h, 1, 2, 4, 1, None) != 0                       # slots 2..5 of 4
    take_log(sim)
    assert sim.b2m_trace_update_predict(c.h, 1, 0, 4, 1, None) == 0, c.err()
    assert [ln.split()[0] for ln in take_log(sim)] == ["trace_update_predict"]
    syncs = c.stats()["host_syncs"]
    assert sim.b2m_run_experts(c.h, 1, T, None) == 0, c.err()                             # consumes the (all-zero) hint matrix
    assert c.stats()["host_syncs"] == syncs + 1
    assert sim.b2m_trace_finish_seq(c.h, 0, None) == 0 and sim.b2m_trace_finish_seq(c.h, 9, None) != 0
    c.close()


def test_random_call_sequences_never_crash_on_cpu(sim, tmp_path, monkeypatch):
    """Stateful fuzz of the C ABI's host logic: random (often invalid) calls in random order.  Every call must return a
    status code (0 or < 0 with a message), the cache invariants must hold after every step, and a valid forward must keep
    working afterwards.  (Run under ASan/UBSan during development: clean.)"""
    rng = np.random.default_rng(2024)
    disk_total = 0
    for trial in range(6):
        Lr, E, k = int(rng.integers(1, 4)), int(rng.choice([2, 4, 8, 16])), 0
        k = int(rng.integers(1, min(E, 4) + 1))
        nslots = int(rng.integers(1, Lr * E + 3))
        chunk = int(rng.choice([0, 4096, 100000]))
        monkeypatch.setenv("B2M_DISK_CHUNK_BYTES", str(int(rng.choice([4096, 12288, 1 << 20]))))
        c = Ctx(sim, L_=Lr, E=E, H=64, I=64, k=k, num_slots=nslots, max_tokens=32, h2d_chunk_bytes=chunk,
                max_inflight_prefetch=int(rng.integers(0, 4)))
        assert c.rc == 0, c.err()
        # a reference-format store holding one blob (3 tensors) per (layer, expert): some experts get registered on it
        import torch
        from moe_infinity_b200.store import ArcherTensorStore
        sdir = tmp_path / f"store{trial}"
        st_ = ArcherTensorStore(str(sdir))
        on_disk = {}
        for l_ in range(Lr):
            for e_ in range(E):
                parts = [rng.integers(0, 255, 64 * 64 * 2, dtype=np.uint8) for _ in range(3)]
                on_disk[(l_, e_)] = np.concatenate(parts)
                for j, p_ in enumerate(parts):
                    st_.store_tensor((l_ * E + e_) * 3 + j, torch.from_numpy(p_), flush=False)
        st_.flush()
        store = C.c_void_p()
        assert sim.b2m_store_open(str(sdir).encode(), 2, 4096, 0, C.byref(store)) == 0
        registered = set()
        reg_count = {}
        nocopy = set()
        x = np.zeros((40, 64), dtype=np.uint16)
        out = np.zeros((40, 64), dtype=np.uint16)
        last_T = None
        for step in range(400):
            op = int(rng.integers(0, 12))
            l = int(rng.integers(-1, Lr + 1))
            e = int(rng.integers(-1, E + 1))
            T = int(rng.integers(0, 36))
            rc = 0
            if op <= 1 and rng.random() < 0.4:
                base = (l * E + e) * 3 if rng.random() < 0.9 else 10 ** 6           # (sometimes ids the store does not have)
                n_ids = 3 if rng.random() < 0.9 else 2
                arr = (C.c_uint32 * 3)(*[(base + j) & 0xFFFFFFFF for j in range(3)])
                rc = sim.b2m_register_expert_on_store(c.h, l, e, store, arr, n_ids)
                if rc == 0:
                    c.blobs[(l, e)] = on_disk[(l, e)]
                    registered.add((l, e))
                    reg_count[(l, e)] = reg_count.get((l, e), 0) + 1
            elif op <= 1:
                blob = rng.integers(0, 255, c.expert_bytes() if rng.random() < 0.9 else 10, dtype=np.uint8)
                rc = sim.b2m_register_expert(c.h, l, e, blob.ctypes.data, blob.nbytes)
                if rc == 0:
                    c.blobs[(l, e)] = blob
                    registered.add((l, e))
                    reg_count[(l, e)] = reg_count.get((l, e), 0) + 1
            elif op <= 4:
                lg = rng.standard_normal((max(T, 1), E)).astype(np.float32)
                rc = sim.b2m_moe_forward(c.h, l, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, out.ctypes.data, None)
                if rc == 0:
                    last_T = T
            elif op == 5:
                lg = rng.standard_normal((max(T, 1), E)).astype(np.float32)
                rc = sim.b2m_route(c.h, l, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None)
                if rc == 0:
                    rc = sim.b2m_run_experts_ex(c.h, l, T, int(rng.choice([1, 2, 3])), None)
            elif op == 6:
                n = int(rng.integers(0, 5))
                pairs = (C.c_int32 * (2 * max(n, 1)))(*[int(v) for _ in range(max(n, 1)) for v in (rng.integers(-1, Lr + 1), rng.integers(-1, E + 1))])
                scores = rng.random(max(n, 1)).astype(np.float32)
                rc = sim.b2m_prefetch_hint(c.h, n, pairs, scores.ctypes.data_as(C.POINTER(C.c_float)))
            elif op == 7:
                rc = sim.b2m_enqueue_prefetch(c.h, l, e)
            elif op == 8:
                rc = sim.b2m_prefetch_drain(c.h) if rng.random() < 0.5 else sim.b2m_prefetch_pump(c.h)
            elif op == 9:
                fl = int(rng.integers(0, 4))
                rc = sim.b2m_make_resident(c.h, l, e, fl, None)
                if rc == 0 and fl & 2:
                    nocopy.add((l, e))                               # slot claimed without a copy: contents are the caller's
            elif op == 10:
                rc = sim.b2m_clear_expert_cache_counts(c.h)
            else:
                rc = sim.b2m_run_experts(c.h, l, T, None)            # usually without a matching routing call
            assert rc <= 0
            if rc != 0:
                assert c.err() != "", (trial, step, op)
            s = c.stats()
            assert s["resident"] <= s["slots"] == min(nslots, Lr * E)      # more slots than experts are not allocated
            assert s["hits"] + s["misses"] == s["dispatches"]
        # residency map and slot contents are consistent after the storm
        seen_slots = {}
        for (l, e) in registered:
            if c.resident(l, e):
                b = c.slot_bytes(l, e)
                assert b is not None
                seen_slots.setdefault(b.ctypes.data, []).append((l, e))
                if reg_count[(l, e)] == 1 and (l, e) not in nocopy:   # registered once (host blob or store): the slot holds those bytes
                    assert np.array_equal(b, c.blobs[(l, e)]), (trial, l, e)
        assert all(len(v) == 1 for v in seen_slots.values()), "two experts share one HBM slot"
        c.close()
        o4 = (C.c_uint64 * 4)()
        assert sim.b2m_store_stats(store, o4) == 0
        disk_total = disk_total + int(o4[0])
        assert sim.b2m_store_close(store) == 0
    assert disk_total > 0, "the fuzz never staged an expert from the store" 
