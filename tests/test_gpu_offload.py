"""GPU: HBM expert cache + prefetch scheduler (forced offload, BASELINE config 3 in miniature).

The CUDA engine must (a) produce the same hidden states as the all-resident run while experts are being
evicted and re-staged from pinned host memory, and (b) reproduce the hit/miss/eviction sequence of
oracle/policy_oracle.py exactly on a seeded routing trace."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import moe_oracle as O  # noqa: E402
from oracle.policy_oracle import CacheOracle  # noqa: E402

H, I, E, K, L = 128, 256, 8, 2, 3
DT = torch.bfloat16


def _model(seed=5):
    experts = [O.make_experts(E, H, I, DT, seed + l, std=0.05) for l in range(L)]
    g = torch.Generator().manual_seed(seed)
    gates = [(torch.randn(E, H, generator=g) * 0.3).to(DT) for _ in range(L)]
    return experts, gates


def _engine(experts, gates, num_slots, **kw):
    from moe_infinity_b200 import MoEEngine
    eng = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=64,
                    num_slots=num_slots, **kw)
    for l in range(L):
        for e in range(E):
            eng.register_expert(l, e, experts[l][e])
        eng.set_gate(l, gates[l])
    return eng


def test_offload_outputs_match_all_resident(lib_built):
    experts, gates = _model()
    full = _engine(experts, gates, L * E)
    small = _engine(experts, gates, 9)            # 9 slots for 24 experts (>= E: one layer's active set must fit)
    g = torch.Generator().manual_seed(1)
    for step in range(6):
        for l in range(L):
            x = torch.randn(7, H, generator=g).to(DT).cuda()
            a = full.forward(l, x)
            b = small.forward(l, x)
            torch.cuda.synchronize()
            assert torch.equal(a, b), f"step {step} layer {l}: offloaded run differs from resident run"
    st = small.stats()
    assert st["misses"] > 0 and st["evictions"] > 0 and st["host_syncs"] == 6 * L
    assert st["h2d_bytes"] == st["misses"] * 3 * H * I * 2
    assert full.stats()["host_syncs"] == 0 and full.stats()["misses"] == 0
    assert st["resident"] <= 9


def test_cache_policy_matches_oracle(lib_built):
    experts, gates = _model(7)
    nslots = 10
    eng = _engine(experts, gates, nslots)
    orc = CacheOracle(L, E, nslots)
    g = torch.Generator().manual_seed(2)
    for step in range(10):
        for l in range(L):
            x = torch.randn(5, H, generator=g).to(DT).cuda()
            before = {e: eng.is_resident(l, e) for e in range(E)}
            eng.forward(l, x)
            counts = eng.last_counts()
            active = [e for e in range(E) if counts[e] > 0]
            exp = orc.dispatch(l, active)
            assert [(e, before[e]) for e in active] == exp, f"step {step} layer {l}"
            for ll in range(L):
                for e in range(E):
                    assert eng.is_resident(ll, e) == orc.resident[ll * E + e]
    s = eng.stats()
    for k in ("dispatches", "hits", "misses", "evictions"):
        assert s[k] == orc.stats[k], k


def test_prefetch_protects_and_counts(lib_built):
    experts, gates = _model(9)
    nslots = 11
    eng = _engine(experts, gates, nslots)
    orc = CacheOracle(L, E, nslots)
    g = torch.Generator().manual_seed(3)
    rng = np.random.default_rng(0)
    for step in range(8):
        for l in range(L):
            x = torch.randn(4, H, generator=g).to(DT).cuda()
            out = eng.forward(l, x)
            counts = eng.last_counts()
            active = [e for e in range(E) if counts[e] > 0]
            orc.dispatch(l, active)
            nl = (l + 1) % L
            cand = rng.choice(E, size=3, replace=False).tolist()
            scores = rng.random(3).tolist()
            pairs = [(nl, int(e)) for e in cand]
            eng.prefetch_hint(pairs, scores)
            eng.prefetch_drain()
            orc.prefetch_hint(pairs, scores)
            for ll in range(L):
                for e in range(E):
                    assert eng.is_resident(ll, e) == orc.resident[ll * E + e], (step, l, ll, e)
    s = eng.stats()
    for k in ("dispatches", "hits", "misses", "evictions", "prefetch_issued", "prefetch_useful"):
        assert s[k] == orc.stats[k], (k, s[k], orc.stats[k])
    assert s["prefetch_issued"] > 0 and s["prefetch_useful"] > 0
    # numerics unaffected by staging order
    ref = _engine(experts, gates, L * E)
    x = torch.randn(9, H, generator=g).to(DT).cuda()
    for l in range(L):
        assert torch.equal(eng.forward(l, x), ref.forward(l, x))


def test_clear_counts_and_chunked_copies(lib_built):
    experts, gates = _model(11)
    eng = _engine(experts, gates, 8, h2d_chunk_bytes=64 * 1024)   # many chunks per expert
    ref = _engine(experts, gates, L * E)
    g = torch.Generator().manual_seed(4)
    for l in range(L):
        x = torch.randn(3, H, generator=g).to(DT).cuda()
        assert torch.equal(eng.forward(l, x), ref.forward(l, x))
    eng.clear_expert_cache_counts()
    assert eng.stats()["misses"] > 0


def test_fewer_slots_than_active_experts_runs_in_waves(lib_built):
    """The reference runs experts one at a time and works with a single slot; here the active set is split into
    waves.  Results and cache statistics must match the all-resident engine / the policy oracle."""
    experts, gates = _model(13)
    ref = _engine(experts, gates, L * E)
    g = torch.Generator().manual_seed(8)
    for nslots in (1, 2, 3):
        eng = _engine(experts, gates, nslots)
        orc = CacheOracle(L, E, nslots)
        for step in range(3):
            for l in range(L):
                x = torch.randn(6, H, generator=g).to(DT).cuda()
                a = eng.forward(l, x)
                b = ref.forward(l, x)
                torch.cuda.synchronize()
                assert torch.equal(a, b), (nslots, step, l)
                counts = eng.last_counts()
                orc.dispatch(l, [e for e in range(E) if counts[e] > 0])
        s = eng.stats()
        for k in ("dispatches", "hits", "misses", "evictions"):
            assert s[k] == orc.stats[k], (nslots, k, s[k], orc.stats[k])


def test_no_evictable_slot_is_an_error_not_an_abort(lib_built):
    from moe_infinity_b200 import B2MError
    experts, gates = _model(13)
    eng = _engine(experts, gates, 2)
    eng.make_resident(1, 0, pin=True)       # both slots pinned by another layer's experts
    eng.make_resident(1, 1, pin=True)
    x = torch.randn(6, H).to(DT).cuda()
    with pytest.raises(B2MError) as ei:
        eng.forward(0, x)
    assert "slot" in str(ei.value)


def test_unregistered_expert_is_an_error(lib_built):
    from moe_infinity_b200 import MoEEngine, B2MError
    eng = MoEEngine(num_layers=1, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=16, num_slots=E)
    eng.set_gate(0, torch.randn(E, H))
    with pytest.raises(B2MError):
        eng.forward(0, torch.randn(4, H).to(DT).cuda())


def test_cache_policy_matches_reference_engine_trace(lib_built):
    """The CUDA engine, driven through the reference-signature `expert_dispatcher` exactly like the reference engine was
    when tests/golden/policy_ref_trace.json was recorded (tools/ref_engine_harness.py --mode policy, protocol
    "sequential"), reproduces the hit flags and resident sets of the reference's real GPUFetchFunc."""
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "policy_ref_trace.json")
    if not os.path.exists(path):
        pytest.skip("golden trace of the reference engine not recorded yet")
    from moe_infinity_b200 import compat
    with open(path) as f:
        g = json.load(f)
    c = g["config"]
    Ln, En, Hn, In, T = c["layers"], c["experts"], c["hidden"], c["inter"], c["tokens"]
    h = compat.prefetch_handle("/tmp/b2m_policy_unused", 0.0)
    d = compat.expert_dispatcher(En, Ln, 0, 4, 8, num_slots=c["slots"], max_tokens=16)
    gen = torch.Generator().manual_seed(c["seed"])
    tid, ids = 0, {}
    for l in range(Ln):
        for e in range(En):
            ids[(l, e)] = list(range(tid, tid + 3))
            for shape in ((In, Hn), (Hn, In), (In, Hn)):
                h.offload((torch.randn(*shape, generator=gen) * 0.05).to(DT), tid)
                tid += 1
            d.register_expert(l, e, ids[(l, e)])
    x = torch.randn(T, Hn, generator=gen).to(DT).cuda()
    cleared = set(g["clear_counts_at"])
    last_n = -1
    for rec in g["sequential"]:
        if rec["n"] != last_n and rec["n"] in cleared:
            d.clear_expert_cache_counts()
        last_n = rec["n"]
        l, e = rec["layer"], rec["expert"]
        act = g["trace"][rec["n"]]["experts"]
        mask = torch.zeros(T, En, dtype=torch.bool)
        for t in range(T):
            mask[t, act[t % len(act)]] = True
            mask[t, act[(t + 1) % len(act)]] = True
        d.set_inputs(x, mask.cuda())
        d.set_expected_queue(1)
        d.enqueue_expert(l, e, 0, False)
        (y, rl, re_, hit), = d.wait_expert()
        assert (rl, re_, int(hit)) == (l, e, rec["hit"]), rec
        res = sorted([ll, ee] for (ll, ee) in ids if d.engine.is_resident(ll, ee))
        assert res == rec["resident_after"], (rec["n"], l, e)


def test_activation_aware_cache_with_lookahead_prefetch(lib_built):
    """B2M_CACHE_ACTIVATION_AWARE + cfg.lookahead_prefetch on the GPU: outputs stay bit-identical to the all-resident run while
    the next layer's experts are staged ahead from this layer's router-logit look-ahead; the look-ahead counts equal the
    top-k of (x @ W_gate[next]^T); the eviction sequence equals oracle/policy_oracle.py (policy 'activation_aware')."""
    from moe_infinity_b200 import MoEEngine, _lib as Lb
    experts, gates = _model(11)
    nslots = 14
    full = _engine(experts, gates, L * E)
    eng = _engine(experts, gates, nslots, cache_policy=Lb.CACHE_ACTIVATION_AWARE, lookahead_prefetch=2, max_inflight_prefetch=4)
    plain = _engine(experts, gates, nslots, cache_policy=Lb.CACHE_ACTIVATION_AWARE)      # same policy, no prefetch: oracle-checkable
    orc = CacheOracle(L, E, nslots, policy="activation_aware")
    g = torch.Generator().manual_seed(2)
    T = 6
    for step in range(8):
        for l in range(L):
            x = torch.randn(T, H, generator=g).to(DT).cuda()
            a = full.forward(l, x)
            b = eng.forward(l, x)
            before = {e: plain.is_resident(l, e) for e in range(E)}
            c = plain.forward(l, x)
            torch.cuda.synchronize()
            assert torch.equal(a, b) and torch.equal(a, c), f"step {step} layer {l}"
            cnt = plain.last_counts()
            active = [e for e in range(E) if cnt[e] > 0]
            assert [(e, before[e]) for e in active] == orc.dispatch(l, active), (step, l)
            # look-ahead = top-k of the next layer's logits on this input (bf16 logits like the Mixtral router; skip near ties)
            look = eng.last_lookahead()
            lg = torch.nn.functional.linear(x.float(), gates[(l + 1) % L].float().cuda())
            top = lg.topk(K + 1, dim=-1).values
            clear = (top[:, K - 1] - top[:, K]) > 0.05 * lg.abs().max()
            if bool(clear.all()):
                want = torch.bincount(lg.topk(K, dim=-1).indices.flatten().cpu(), minlength=E).tolist()
                assert look == want, (step, l)
    st = eng.stats()
    assert st["prefetch_issued"] > 0 and st["prefetch_useful"] > 0
    assert st["host_syncs"] == 8 * L                       # the look-ahead rides on the per-layer count read-back
    for ll in range(L):
        for e in range(E):
            assert plain.is_resident(ll, e) == orc.resident[ll * E + e]


def test_disk_backed_experts_match_host_backed(lib_built, tmp_path, monkeypatch):
    """SURVEY §8f N3, the disk tier: half of the experts stay on a reference-format store (written by store.py) and are
    staged disk -> pinned chunk ring -> HBM slot on a miss (b2m_register_expert_on_store; reader: csrc/store_reader.cpp);
    the hidden states must equal the all-resident run bit for bit and the cache bookkeeping must not notice the difference."""
    from moe_infinity_b200.store import ArcherTensorStore, NativeStoreReader
    monkeypatch.setenv("B2M_DISK_CHUNK_BYTES", str(10 * 4096))        # 196608-byte blobs: 5 chunks, crossing tensor ends
    experts, gates = _model(21)
    full = _engine(experts, gates, L * E)
    host = _engine(experts, gates, 9)
    st = ArcherTensorStore(str(tmp_path))
    ids, tid = {}, 1000
    for l in range(L):
        for e in range(0, E, 2):
            ids[(l, e)] = list(range(tid, tid + 3))
            for w in experts[l][e]:                                     # (w1, w2, w3) in blob order
                st.store_tensor(tid, w, flush=False)
                tid += 1
    st.flush()
    rd = NativeStoreReader(str(tmp_path), num_threads=4, block_bytes=16384)
    from moe_infinity_b200 import MoEEngine
    disk = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=64, num_slots=9)
    for l in range(L):
        for e in range(E):
            if (l, e) in ids:
                disk.register_expert_on_store(l, e, rd, ids[(l, e)])
            else:
                disk.register_expert(l, e, experts[l][e])
        disk.set_gate(l, gates[l])
    g = torch.Generator().manual_seed(4)
    for step in range(6):
        for l in range(L):
            x = torch.randn(7, H, generator=g).to(DT).cuda()
            a, b, c = full.forward(l, x), host.forward(l, x), disk.forward(l, x)
            torch.cuda.synchronize()
            assert torch.equal(a, c), f"step {step} layer {l}: disk-backed run differs from the resident run"
            assert torch.equal(b, c)
    sh, sd = host.stats(), disk.stats()
    for k in ("dispatches", "hits", "misses", "evictions", "h2d_bytes"):
        assert sh[k] == sd[k], k
    assert sd["misses"] > 0 and sd["evictions"] > 0
    rs = rd.stats()
    assert rs["bytes_read"] > 0 and rs["bytes_read"] % (3 * H * I * 2) == 0
    del disk
    rd.close()
