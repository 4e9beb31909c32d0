"""CPU: the rows of tests/ep_loopback.py, before any of them costs GPU time.

* Coverage: the table reaches 2, 4, 8 and 16 ranks, 1 and 128 experts per rank, both counts layouts, both 16-bit dtypes, an
  owner whose down GEMM runs split-K and one that runs whole-K (the plan api.cu logs on the host simulation), more than 256
  tokens per owner, a rank without tokens, a rank that receives nothing, a full peer segment, dropped tokens, a shared
  expert and every router kind whose ROUTERS row in api.cu allows expert parallelism.
* Pre-flight: every row's call sequence, with the GPU test's capacity, max_tokens, buffer layout and router inputs, returns
  B2M_OK on the host simulation (tests/host/sim, relinked with ep_probe.cpp, which refuses what ep.cu's launchers refuse
  and records each exchange launch); regroup clears y whenever the owner's down GEMM runs split-K, the return trip keeps
  the pack's counts layout, and the inline layout past 4E = 2H and an fp32-numerics context are refused.
* expected_exchange agrees with a per-token restatement of ep.cu's exchange contract on random routings with dropped
  (-1) entries."""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
import ep_loopback as EP  # noqa: E402
import gemm_exact_cases as X  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402

_DT = {"bf16": L.DTYPE_BF16, "f16": L.DTYPE_F16}
_OBJS = ("api.o", "fake_kernels.o", "fake_cudart.o", "store_reader.o")
_WRAPPED = ("_ZN3b2m14launch_ep_packERKNS_8EpParamsEiP11CUstream_st", "_ZN3b2m17launch_ep_regroupERKNS_8EpParamsEP11CUstream_st",
            "_ZN3b2m17launch_ep_ungroupERKNS_8EpParamsEiP11CUstream_st",
            "_ZN3b2m16launch_ep_unpackERKNS_8EpParamsEiiP11CUstream_st")


# ------------------------------------------------------------------------------------------------ host simulation
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    """The host simulation's objects relinked with tests/host/sim/ep_probe.cpp (-Wl,--wrap on the four exchange
    launchers), which refuses what ep.cu's launchers refuse and records each launch's geometry and y_zero count."""
    so = build_sim.build()
    if so is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    objs = [os.path.join(build_sim.OUT, n) for n in _OBJS]
    if not all(os.path.exists(o) for o in objs):     # objects of an older build removed: build the simulation afresh
        os.remove(so)
        build_sim.build()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(build_sim._nvcc())), "include")
    inc = ["-I", build_sim.CSRC, "-I", os.path.join(build_sim.ROOT, "include"), "-I", cuda_inc]
    out = tmp_path_factory.mktemp("ep_probe")
    obj, so = str(out / "ep_probe.o"), str(out / "libb2m_hostsim_ep.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", *inc, "-c", os.path.join(HERE, "host", "sim", "ep_probe.cpp"),
                    "-o", obj], check=True, capture_output=True)
    subprocess.run(["g++", "-shared", "-Wl,-Bsymbolic", *[f"-Wl,--wrap={w}" for w in _WRAPPED], "-o", so, *objs, obj,
                    "-lpthread"], check=True, capture_output=True)
    lib = C.CDLL(so)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.b2m_sim_take_log.restype, lib.b2m_sim_take_log.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t]
    lib.b2m_probe_take_ep.restype, lib.b2m_probe_take_ep.argtypes = C.c_size_t, [C.POINTER(C.c_int64), C.c_size_t]
    return lib


def _take_log(lib):
    buf = C.create_string_buffer(1 << 22)
    assert lib.b2m_sim_take_log(buf, len(buf)) < len(buf)
    return [ln for ln in buf.value.decode().split("\n") if ln]


def _kv(line):
    return {m.group(1): m.group(2) for m in re.finditer(r"(\w+)=(\[[^\]]*\]|\S+)", line)}


_EP_KIND = ("pack", "regroup", "ungroup", "unpack")


def _take_ep(lib):
    """The exchange launches since the last call: dicts of kind, nranks, rank, cap, inline, y_zero."""
    buf = (C.c_int64 * 6144)()
    n = lib.b2m_probe_take_ep(buf, len(buf))
    assert n <= len(buf)
    return [dict(kind=_EP_KIND[buf[i]], nranks=buf[i + 1], rank=buf[i + 2], cap=buf[i + 3], inline=buf[i + 4],
                 y_zero=buf[i + 5]) for i in range(0, n, 6)]


class SimRank:
    """One simulated rank: the context tests/test_gpu_ep_loopback.py creates, with zero-filled host blobs for its experts."""

    def __init__(self, lib, c: EP.EpCase, rank: int, numerics: int = L.NUMERICS_REFERENCE):
        self.lib, self.c = lib, c
        E, H = c.E, c.H
        cfg = L.Config()
        cfg.struct_size = C.sizeof(L.Config)
        cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = c.layers, E, H, c.I, c.k
        cfg.dtype, cfg.expert_type, cfg.router = _DT[c.dtype], X.ETYPE[c.etype], EP.ROUTER_ID[c.router]
        cfg.gate_dtype = _DT[c.dtype] if c.router == EP.MIXTRAL else L.DTYPE_F32
        cfg.numerics, cfg.max_tokens, cfg.num_slots = numerics, c.max_tokens, c.layers * (E // c.N)
        cfg.shared_inter, cfg.n_group, cfg.topk_group = c.shared, c.n_group, c.topk_group
        cfg.expert_capacity, cfg.routed_scaling_factor = c.expert_capacity, 1.0
        self.h = C.c_void_p()
        assert lib.b2m_ctx_create(C.byref(cfg), C.byref(self.h)) == 0, self.err()
        s = L.Stats()
        assert lib.b2m_stats_get(self.h, C.byref(s)) == 0
        self.blob = np.zeros(s.as_dict()["slot_bytes"], dtype=np.uint8)
        self.keep = [self.blob]
        El = E // c.N
        for l in range(c.layers):
            for e in range(rank * El, (rank + 1) * El):
                assert lib.b2m_register_expert(self.h, l, e, self.blob.ctypes.data, self.blob.nbytes) == 0, self.err()
                assert lib.b2m_make_resident(self.h, l, e, 1, None) == 0, self.err()
            if c.shared:
                sh = np.zeros(3 * H * c.shared * 2, dtype=np.uint8)
                self.keep.append(sh)
                assert lib.b2m_register_shared(self.h, l, sh.ctypes.data, sh.nbytes) == 0, self.err()
            if c.router == EP.V3:
                bias = np.zeros(E, dtype=np.float32)
                self.keep.append(bias)
                assert lib.b2m_set_gate_bias(self.h, l, bias.ctypes.data) == 0, self.err()

    def err(self):
        return (self.lib.b2m_last_error(self.h) or b"").decode()

    def close(self):
        self.lib.b2m_ctx_destroy(self.h)

    def route(self, layer, T, lg, sc):
        x = np.zeros((max(T, 1), self.c.H), dtype=np.uint16)
        rin, kind = (lg, 1) if sc is None else (sc, 2)
        rin = np.ascontiguousarray(rin.numpy(), dtype=np.float32)
        seq = T if self.c.router == EP.SWITCH else 0
        # a rank without tokens hands over null pointers, as torch does for an empty tensor
        ptr = (lambda a: a.ctypes.data) if T else (lambda a: None)
        return self.lib.b2m_route(self.h, layer, ptr(x), ptr(rin), kind, L.DTYPE_F32, T, seq, None)


def sim_step(lib, c: EP.EpCase, ranks, step: int, layout: str):
    """One step of the row on the simulated ranks, every call asserted B2M_OK; -> per layer, per owner, the K4 ksplit and
    the regroup's y_zero count."""
    N, H, cap, Ts = c.N, c.H, c.capacity, c.steps[step]
    rows = cap + 1 if layout == EP.INLINE else cap
    bufs = np.zeros((N, N, rows, H), dtype=np.uint16)
    cnt = np.zeros((N, N, c.E), dtype=np.int32)
    sep = layout == EP.SEPARATE
    plans = []
    _take_ep(lib)
    for l in range(c.layers):
        for r, rk in enumerate(ranks):
            lg, sc = EP.router_input(c, l, r, Ts[r], seed=100 * step + 10 * l + r)
            assert rk.route(l, Ts[r], lg, sc) == 0, (c.name, r, rk.err())
        for r, rk in enumerate(ranks):
            assert lib.b2m_ep_pack(rk.h, N, r, cap, Ts[r], bufs[r].ctypes.data, cnt[r, 0].ctypes.data if sep else None,
                                   None) == 0, (c.name, r, rk.err())
        _take_log(lib)
        packs = _take_ep(lib)
        assert [(p["kind"], p["rank"], p["inline"]) for p in packs] == [("pack", r, int(not sep)) for r in range(N)]
        for r, rk in enumerate(ranks):
            assert lib.b2m_ep_regroup(rk.h, N, r, cap, sum(Ts), bufs[r].ctypes.data, cnt[r].ctypes.data if sep else None,
                                      None) == 0, (c.name, r, rk.err())
        _take_log(lib)
        regroups = _take_ep(lib)
        assert [(p["kind"], p["rank"], p["cap"]) for p in regroups] == [("regroup", r, cap) for r in range(N)]
        zero = [p["y_zero"] for p in regroups]
        layer_plans = []
        for r, rk in enumerate(ranks):
            assert lib.b2m_run_experts(rk.h, l, sum(Ts), None) == 0, (c.name, r, rk.err())
            dn = [_kv(ln) for ln in _take_log(lib) if ln.startswith("gemm") and _kv(ln)["epi"] == "1"]
            assert len(dn) == 1, (c.name, r, dn)
            layer_plans.append((int(dn[0]["ksplit"]), zero[r]))
        for r, rk in enumerate(ranks):
            assert lib.b2m_ep_ungroup(rk.h, N, r, cap, bufs[r].ctypes.data, None) == 0, (c.name, r, rk.err())
            assert lib.b2m_ep_unpack(rk.h, N, r, cap, Ts[r], bufs[r].ctypes.data, None) == 0, (c.name, r, rk.err())
            x = np.zeros((max(Ts[r], 1), H), dtype=np.uint16)
            out = np.zeros_like(x)
            assert lib.b2m_combine(rk.h, l, x.ctypes.data, Ts[r], out.ctypes.data, None) == 0, (c.name, r, rk.err())
        # the return trip runs in the layout the pack chose
        assert [(p["kind"], p["rank"], p["inline"]) for p in _take_ep(lib)] == \
            [(k, r, int(not sep)) for r in range(N) for k in ("ungroup", "unpack")]
        plans.append(layer_plans)
    return plans


_PLANS = {}


def row_plans(lib, c: EP.EpCase):
    """(step, layer, rank) -> (ksplit of the owner's down GEMM, floats regroup clears) for every step of the row."""
    if c.name not in _PLANS:
        ranks = [SimRank(lib, c, r) for r in range(c.N)]
        try:
            _PLANS[c.name] = {(s, l, r): p for s in range(len(c.steps))
                              for l, lp in enumerate(sim_step(lib, c, ranks, s, c.layout(s))) for r, p in enumerate(lp)}
        finally:
            for rk in ranks:
                rk.close()
    return _PLANS[c.name]


@pytest.mark.parametrize("name", [c.name for c in EP.CASES])
def test_row_call_sequence_runs_on_the_host_simulation(sim, name):
    c = EP.BY_NAME[name]
    plans = row_plans(sim, c)
    for (s, l, r), (ksplit, zeroed) in plans.items():
        # split-K accumulates into y with atomics: regroup must clear every row the owner's GEMM may write
        if ksplit > 1:
            assert zeroed == c.N * c.capacity * c.H, (name, s, l, r, ksplit, zeroed)
    print(name, sorted(set(p[0] for p in plans.values())))


def test_refusals_on_the_host_simulation(sim):
    """The inline layout needs 4E <= 2H (E=256, H=256 is refused, the context then runs the separate layout); fp32
    numerics are refused by every expert-parallel entry point (the exchange returns model-dtype rows, the single-GPU fp32
    combine reads unrounded fp32 outputs)."""
    c = EP.BY_NAME["e256_n2_el128"]
    wide = EP.EpCase("e256_h256", EP.GREEDY, 256, 512, 256, 8, "bf16", 2, ((16, 16),), (EP.SEPARATE,), "refusal",
                     design=c.design)
    ranks = [SimRank(sim, wide, r) for r in range(2)]
    try:
        lg, sc = EP.router_input(wide, 0, 0, 16, seed=1)
        assert ranks[0].route(0, 16, lg, sc) == 0
        rows = np.zeros((2, wide.capacity + 1, wide.H), dtype=np.uint16)
        assert sim.b2m_ep_pack(ranks[0].h, 2, 0, wide.capacity, 16, rows.ctypes.data, None, None) != 0
        assert sim.b2m_ep_regroup(ranks[0].h, 2, 0, wide.capacity, 32, rows.ctypes.data, None, None) != 0
        sim_step(sim, wide, ranks, 0, EP.SEPARATE)
    finally:
        for rk in ranks:
            rk.close()
    m = EP.BY_NAME["mixtral_n8_el1"]
    small = EP.EpCase("fp32num", EP.MIXTRAL, 256, 512, 8, 2, "bf16", 2, ((4, 4),), (EP.INLINE,), "refusal")
    for cc in (small, m):
        rk = SimRank(sim, cc, 0, numerics=L.NUMERICS_FP32)
        try:
            cap, N = cc.capacity, cc.N
            rows = np.zeros((N, cap + 1, cc.H), dtype=np.uint16)
            lg, sc = EP.router_input(cc, 0, 0, cc.steps[0][0], seed=2)
            assert rk.route(0, cc.steps[0][0], lg, sc) == 0
            p = rows.ctypes.data
            for rc in (sim.b2m_ep_pack(rk.h, N, 0, cap, cc.steps[0][0], p, None, None),
                       sim.b2m_ep_regroup(rk.h, N, 0, cap, sum(cc.steps[0]), p, None, None),
                       sim.b2m_ep_ungroup(rk.h, N, 0, cap, p, None),
                       sim.b2m_ep_unpack(rk.h, N, 0, cap, cc.steps[0][0], p, None),
                       sim.b2m_ep_p2p_init(rk.h, N, 0, cap, (C.c_char * 64)())):
                assert rc == L.B2M_EUNSUPPORTED and "fp32" in rk.err(), (rc, rk.err())
            assert sim.b2m_ep_p2p_dispatch(rk.h, cc.steps[0][0], None) != 0           # never initialised
        finally:
            rk.close()


# ------------------------------------------------------------------------------------------------ coverage
def _ep_routers():
    """Names of the router kinds whose ROUTERS row in api.cu allows expert parallelism."""
    src = open(os.path.join(build_sim.CSRC, "api.cu")).read()
    rows = re.findall(r'\{B2M_ROUTER_\w+,\s*"(\w+)",[^}]*?\b(true|false),\s*COMBINE_\w+,\s*COMBINE_\w+\}', src)
    assert len(rows) == 7, rows
    return {n for n, ep in rows if ep == "true"}


def _designed_layers(c):
    """(step, layer, per-rank counts) of the row's designed routings."""
    for s, Ts in enumerate(c.steps):
        for l in range(c.layers):
            yield s, l, [c.design(l, r, T, c.E, c.k) for r, T in enumerate(Ts)]


def coverage(plans=None):
    cov = {}

    def add(item, name):
        cov.setdefault(item, []).append(name)
    for c in EP.CASES:
        add(f"N={c.N}", c.name)
        add(f"El={c.El}", c.name)
        for lay in c.layouts:
            add(f"layout {lay}", c.name)
        add(f"dtype {c.dtype}", c.name)
        add(f"router {c.router}", c.name)
        if max(sum(Ts) for Ts in c.steps) > 256:
            add("T_total > 256", c.name)
        if any(0 in Ts for Ts in c.steps):
            add("a rank without tokens", c.name)
        if c.shared:
            add("a shared expert", c.name)
        if c.expert_capacity:
            add("dropped tokens", c.name)
        if c.design is not None:
            for s, l, cnts in _designed_layers(c):
                routed = [sum(x[e] for x in cnts) for e in range(c.E)]
                if any(sum(routed[r * c.El:(r + 1) * c.El]) == 0 for r in range(c.N)):
                    add("a rank that receives nothing", c.name)
                if 0 in routed:
                    add("an expert no rank routes to", c.name)
                for r, x in enumerate(cnts):
                    per_owner = [sum(x[o * c.El:(o + 1) * c.El]) for o in range(c.N)]
                    if c.capacity in per_owner:
                        add("a full peer segment", c.name)
        if plans is not None:
            for (ks, _) in plans[c.name].values():
                add("owner split-K" if ks > 1 else "owner whole-K", c.name)
    return cov


def test_rows_cover_the_exchange(sim):
    plans = {c.name: row_plans(sim, c) for c in EP.CASES}
    cov = coverage(plans)
    required = ([f"N={n}" for n in (2, 4, 8, 16)] + ["El=1", "El=128", "layout inline", "layout separate", "dtype bf16",
                "dtype f16", "owner split-K", "owner whole-K", "T_total > 256", "a rank without tokens",
                "a rank that receives nothing", "an expert no rank routes to", "a full peer segment", "dropped tokens",
                "a shared expert"] + [f"router {n}" for n in sorted(_ep_routers())])
    for item in required:
        print(f"{item:32s} {', '.join(sorted(set(cov.get(item, [])))) or '-- MISSING'}")
    assert not [i for i in required if not cov.get(i)]
    assert _ep_routers() == {EP.MIXTRAL, EP.GREEDY, EP.GROUP, EP.SWITCH, EP.V3}
    assert "mixtral_full_n2_t1" in cov["owner split-K"]


def test_designed_routings_are_valid():
    """Each designed routing has k distinct experts per token, no expert above T_local, no ties at the k-th choice, and
    its logits rank exactly the designed experts first."""
    for c in EP.CASES:
        if c.design is None:
            continue
        for s, l, cnts in _designed_layers(c):
            for r, (T, x) in enumerate(zip(c.steps[s], cnts)):
                assert len(x) == c.E and sum(x) == T * c.k and max(x) <= T, (c.name, s, l, r)
                if T == 0:
                    continue
                lg, sc = EP.router_input(c, l, r, T, seed=0)
                v = (lg if sc is None else sc)[:T]
                top = torch.sort(v, dim=-1, descending=True).values
                assert bool((top[:, c.k - 1] > top[:, c.k]).all()), (c.name, s, l, r)
                idx = torch.topk(v, c.k, dim=-1).indices
                assert torch.equal(torch.bincount(idx.flatten(), minlength=c.E), torch.tensor(x)), (c.name, s, l, r)


# ------------------------------------------------------------------------------------------------ expected_exchange
def _brute(topk, N, E):
    """The contract token by token: owner r's rows are, for each of its experts e in turn, for each source s in turn,
    the tokens t of s that chose e in ascending order; the slot of (s, t, e) in s's segment for r counts the (t', e')
    of s bound for r that sort before it by expert, then token."""
    El = E // N
    lists = [t.tolist() for t in topk]

    def before(s, r, e, t):
        return sum(1 for t2, row in enumerate(lists[s]) for e2 in row
                   if e2 >= 0 and e2 // El == r and (e2 < e or (e2 == e and t2 < t)))
    out = []
    for r in range(N):
        tok, sl = [], []
        for e in range(r * El, (r + 1) * El):
            for s in range(N):
                for t, row in enumerate(lists[s]):
                    if e in row:
                        tok.append((s, t))
                        sl.append((s, before(s, r, e, t)))
        send = [[t for e in range(r * El, (r + 1) * El) for t, row in enumerate(lists[s]) if e in row] for s in range(N)]
        offs = [sum(1 for e2 in range(r * El, (r + 1) * El) for s in range(N) for row in lists[s] if e2 < e and e2 in row)
                for e in range(E + 1)]
        out.append((tok, sl, send, offs))
    return out


@pytest.mark.parametrize("N,E,k", [(2, 8, 2), (4, 8, 1), (4, 64, 6), (8, 64, 6), (16, 64, 3)])
def test_expected_exchange_is_the_contract(N, E, k):
    g = torch.Generator().manual_seed(N * 100 + E + k)
    for trial in range(4):
        topk = []
        for s in range(N):
            T = int(torch.randint(0, 9, (1,), generator=g))
            idx = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]) if T else torch.zeros(0, k, dtype=torch.int64)
            drop = torch.rand(idx.shape, generator=g) < 0.2
            topk.append(torch.where(drop, torch.full_like(idx, -1), idx))
        ex = EP.expected_exchange(topk, N, E)
        want = _brute(topk, N, E)
        for r, (tok, sl, send, offs) in enumerate(want):
            assert ex.token[r] == tok and ex.slot[r] == sl and ex.offsets[r] == offs, (N, E, k, trial, r)
            assert [ex.send[s][r] for s in range(N)] == send
        for s in range(N):
            assert ex.counts[s] == torch.bincount(topk[s][topk[s] >= 0].flatten(), minlength=E).tolist()
