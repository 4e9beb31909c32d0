"""GPU, one device: the expert-parallel exchange kernels of csrc/ep.cu (pack, regroup, ungroup, unpack) with every rank in
one process (tests/ep_loopback.py), exact against a float64 reference on every row of ep_loopback.CASES.

The experts are the integer data of tests/gemm_exact_cases.py, so every partial sum is exact in fp32 and every comparison is
torch.equal, whatever split-K plan an owner picks.  After each phase of each layer:
* pack: every peer segment holds exactly the source's rows bound for that peer, slots past the count keep the NaN
  sentinel, and the counts (the inline counts row, or send_counts) are the source's;
* regroup: the owner's offsets over global expert ids and its gathered rows are expected_exchange's, bit for bit;
* run_experts + ungroup: the owner's hmid and y are the reference, every filled return slot holds y in the model dtype and
  every other slot keeps the sentinel;
* unpack: the source's y holds the returned rows at its own permuted row positions;
* combine: the layer output equals the oracle combine replayed on the engine's routing (Mixtral and DeepSeek rows) and,
  bit for bit, a single engine holding all E experts run on the same rank's tokens; no host synchronisation.
Plus a CUDA graph of a whole two-layer step, and the refusals (inline counts past 4E = 2H, fp32 numerics).
The peer-to-peer exchange (b2m_ep_p2p_*) needs CUDA IPC between processes and is checked by tests/test_gpu_ep.py."""
from __future__ import annotations

import pytest
import torch

import ep_loopback as EP
import gemm_exact_cases as X
from test_gpu_gemm_exact import _replay_combine, _same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def live():
    """Every engine a test of this module creates; all closed when the module ends."""
    held = []
    yield held
    for h in held:
        h.close()
    held.clear()
    torch.cuda.empty_cache()


def _release(live):
    for h in live:
        h.close()
    live.clear()
    torch.cuda.empty_cache()


def _data(c: EP.EpCase):
    ec = c.expert_case()
    experts = [[X.make_expert(ec, seed=1000 * l + e + 1, dev="cuda") for e in range(c.E)] for l in range(c.layers)]
    shared = [X.make_expert(c.shared_case(), seed=999 - l, dev="cuda") for l in range(c.layers)] if c.shared else None
    g = torch.Generator().manual_seed(5)
    bias = [torch.randn(c.E, generator=g) * 0.5 for _ in range(c.layers)] if c.router == EP.V3 else None
    return experts, shared, bias


def _engine(c: EP.EpCase, data, rank, numerics=None):
    """Rank `rank`'s context (its own experts only), or with rank None a single context holding all E experts."""
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    experts, shared, bias = data
    mine = range(c.E) if rank is None else range(rank * c.El, (rank + 1) * c.El)
    eng = MoEEngine(num_layers=c.layers, num_experts=c.E, hidden=c.H, inter=c.I, top_k=c.k, dtype=X.DTYPES[c.dtype],
                    expert_type=X.ETYPE[c.etype], router=EP.ROUTER_ID[c.router],
                    numerics=L.NUMERICS_REFERENCE if numerics is None else numerics, max_tokens=c.max_tokens,
                    num_slots=c.layers * len(mine), shared_inter=c.shared, n_group=c.n_group, topk_group=c.topk_group,
                    expert_capacity=c.expert_capacity, pack_weights=rank is not None)
    for l in range(c.layers):
        for e in mine:
            eng.load_expert(l, e, experts[l][e].load)
        if shared:
            eng.register_shared(l, shared[l].w)
        if bias:
            eng.set_gate_bias(l, bias[l])
    return eng


def _inputs(c: EP.EpCase, step: int, layer: int):
    xs = [X.make_x(T, c.H, X.DTYPES[c.dtype], seed=7919 * step + 101 * layer + r, dev="cuda")
          for r, T in enumerate(c.steps[step])]
    rins = []
    for r, T in enumerate(c.steps[step]):
        lg, sc = EP.router_input(c, layer, r, T, seed=100 * step + 10 * layer + r)
        rins.append((None if lg is None else lg.cuda(), None if sc is None else sc.cuda()))
    return xs, rins


def _sentinel_rows(t: torch.Tensor) -> bool:
    return bool((t.view(torch.int16) == EP.SENTINEL).all())


class Checker:
    """probe(phase) of LoopbackEP.layer: checks every rank's state after that phase against the expected exchange and the
    float64 reference."""

    def __init__(self, c: EP.EpCase, lb: EP.LoopbackEP, data, xs, layout, cap, layer):
        self.c, self.lb, self.xs, self.layout, self.cap, self.layer = c, lb, xs, layout, cap, layer
        self.experts, self.shared, _ = data
        self.Ts = [x.shape[0] for x in xs]
        self.dt = X.DTYPES[c.dtype]
        self.rins = None
        self.dropped = 0

    def __call__(self, phase):
        torch.cuda.synchronize()
        getattr(self, phase)()

    def pack(self):
        c, lb, N = self.c, self.lb, self.c.N
        self.topk = [e.ws("topk_idx", T).long().cpu() for e, T in zip(lb.engines, self.Ts)]
        self.dropped = sum(int((t < 0).sum()) for t in self.topk)
        ex = self.ex = EP.expected_exchange(self.topk, N, c.E)
        b = lb.buffers(self.layout, self.cap)
        for s in range(N):
            if c.design is not None and self.Ts[s]:
                want = c.design(self.layer, s, self.Ts[s], c.E, c.k)
                assert lb.engines[s].ws("counts", self.Ts[s]).tolist() == list(want), (c.name, s, "routing is not the design")
            # the source's permuted rows are its (expert, token) pairs in expert-major, token order
            row_of = lb.engines[s].ws("row_of", self.Ts[s]).long().cpu()
            pairs = sorted((int(e), t) for t, row in enumerate(self.topk[s].tolist()) for e in row if e >= 0)
            pos = {p: i for i, p in enumerate(pairs)}
            for t in range(self.Ts[s]):
                for j in range(c.k):
                    e = int(self.topk[s][t, j])
                    assert int(row_of[t, j]) == (pos[(e, t)] if e >= 0 else -1), (c.name, s, t, j)
            for r in range(N):
                seg, toks = b["send"][s][r], ex.send[s][r]
                _same(seg[:len(toks)], self.xs[s][torch.tensor(toks, dtype=torch.long, device="cuda")],
                      f"{c.name} send {s}->{r}")
                assert _sentinel_rows(seg[len(toks):self.cap]), f"{c.name} send {s}->{r}: a slot past the count was written"
                if self.layout == EP.INLINE:
                    row = seg[self.cap].view(torch.int16)
                    assert row[:2 * c.E].view(torch.int32).tolist() == ex.counts[s], f"{c.name} inline counts {s}->{r}"
                    assert bool((row[2 * c.E:] == EP.SENTINEL).all()), f"{c.name} counts row {s}->{r} past E"
            if self.layout == EP.SEPARATE:
                assert b["send_counts"][s].tolist() == ex.counts[s], f"{c.name} send_counts of {s}"

    def regroup(self):
        c, ex = self.c, self.ex
        T_total = sum(self.Ts)
        for r, e in enumerate(self.lb.engines):
            assert e.ws("offsets", T_total).tolist() == ex.offsets[r], f"{c.name} owner {r} offsets"
            n = len(ex.token[r])
            if n:
                want = torch.stack([self.xs[s][t] for s, t in ex.token[r]])
                _same(e.ws("xp", T_total)[:n], want, f"{c.name} owner {r} xp")

    def ungroup(self):
        c, ex, N = self.c, self.ex, self.c.N
        T_total = sum(self.Ts)
        ec = c.expert_case()
        b = self.lb.buffers(self.layout, self.cap)
        self.y_of = {}                                         # (source, token, expert) -> reference y row
        for r, e in enumerate(self.lb.engines):
            n = len(ex.token[r])
            hmid, y = e.ws("hmid", T_total), e.ws("y", T_total)
            y_ref = torch.empty(n, c.H, dtype=torch.float32, device="cuda")
            for g in range(r * c.El, (r + 1) * c.El):
                r0, r1 = ex.offsets[r][g], ex.offsets[r][g + 1]
                if r0 == r1:
                    continue
                x = torch.stack([self.xs[s][t] for s, t in ex.token[r][r0:r1]])
                h_ref, y_ref[r0:r1] = X.reference(ec, x, self.experts[self.layer][g].w)
                _same(hmid[r0:r1], h_ref, f"{c.name} owner {r} expert {g} hmid")
                _same(y[r0:r1], y_ref[r0:r1], f"{c.name} owner {r} expert {g} y")
            for i, ((s, t), g) in enumerate(zip(ex.token[r], ex.expert[r])):
                self.y_of[(s, t, g)] = y_ref[i]
            for s in range(N):
                idx = [i for i, (s2, _) in enumerate(ex.slot[r]) if s2 == s]
                slots = [ex.slot[r][i][1] for i in idx]
                assert slots == list(range(len(slots))), (c.name, r, s, slots)
                seg = b["ret"][r][s]
                if idx:
                    _same(seg[:len(idx)], y_ref[torch.tensor(idx, device="cuda")].to(self.dt), f"{c.name} ret {r}->{s}")
                assert _sentinel_rows(seg[len(idx):]), f"{c.name} ret {r}->{s}: a slot past the count was written"

    def unpack(self):
        c = self.c
        self.y_src = []
        for s, e in enumerate(self.lb.engines):
            T = self.Ts[s]
            want = torch.zeros(T * c.k, c.H, dtype=torch.float32, device="cuda")
            row_of = e.ws("row_of", T).long().cpu()
            n = 0
            for t in range(T):
                for j in range(c.k):
                    g = int(self.topk[s][t, j])
                    if g >= 0:
                        want[int(row_of[t, j])] = self.y_of[(s, t, g)].to(self.dt).float()
                        n += 1
            _same(e.ws("y", T)[:n], want[:n], f"{c.name} source {s} y after unpack")
            self.y_src.append(want)

    def combine(self):
        c = self.c
        self.checked_oracle = 0
        if c.router not in (EP.MIXTRAL, EP.GREEDY, EP.GROUP):
            return
        for r, e in enumerate(self.lb.engines):
            T = self.Ts[r]
            if T == 0:
                continue
            rc = X.Case(c.name, c.etype, c.H, c.I, c.E, c.k, c.dtype, "bf16", T, (T * c.k,), X.Plan(0, 0, *[False] * 5))
            y_sh = X.reference(c.shared_case(), self.xs[r], self.shared[self.layer].w)[1] if c.shared else None
            _same(self.outs[r].reshape(T, c.H), _replay_combine(rc, e, self.y_src[r], y_sh), f"{c.name} rank {r} output")
            self.checked_oracle += 1


def _single(c, single, layer, x, rin):
    lg, sc = rin
    T = x.shape[0]
    return single.forward(layer, x, router_logits=None if lg is None else lg[:T], scores=None if sc is None else sc[:T],
                          seq_len=T if c.router == EP.SWITCH else 0)


def run_row(c: EP.EpCase, lb: EP.LoopbackEP, single, data, steps=None):
    """Every step of the row with the phase checks; -> number of rows dropped by the routing over all steps."""
    dropped = 0
    for s in (range(len(c.steps)) if steps is None else steps):
        layout, cap = c.layout(s), c.capacity
        for l in range(c.layers):
            xs, rins = _inputs(c, s, l)
            outs = [torch.empty(x.shape[0], c.H, dtype=x.dtype, device="cuda") for x in xs]
            chk = Checker(c, lb, data, xs, layout, cap, l)
            chk.outs = outs
            syncs0 = [e.stats()["host_syncs"] for e in lb.engines]
            lb.fill_sentinels(lb.buffers(layout, cap))
            lb.layer(l, xs, rins, outs, layout, cap, probe=chk)
            torch.cuda.synchronize()
            assert [e.stats()["host_syncs"] for e in lb.engines] == syncs0, f"{c.name}: a host synchronisation in the step"
            dropped += chk.dropped
            for r, x in enumerate(xs):
                if x.shape[0]:
                    _same(outs[r], _single(c, single, l, x, rins[r]).reshape(outs[r].shape),
                          f"{c.name} step {s} layer {l} rank {r}: expert-parallel vs single engine")
    return dropped


@pytest.mark.parametrize("name", [c.name for c in EP.CASES])
def test_exchange_is_exact(lib_built, live, name):
    _release(live)
    c = EP.BY_NAME[name]
    data = _data(c)
    lb = EP.LoopbackEP(c, lambda r: _engine(c, data, r))
    live.append(lb)
    single = _engine(c, data, None)
    live.append(single)
    dropped = run_row(c, lb, single, data)
    assert (dropped > 0) == (c.expert_capacity > 0), (name, dropped)
    _release(live)


def test_graph_capture_of_a_step(lib_built, live):
    """One two-layer step of mixtral_n8_el1 -- every rank's calls and the exchange copies -- captured in a CUDA graph and
    replayed with new inputs written in place: each replay equals the eager step and the single engine."""
    _release(live)
    c = EP.BY_NAME["mixtral_n8_el1"]
    data = _data(c)
    lb = EP.LoopbackEP(c, lambda r: _engine(c, data, r))
    live.append(lb)
    single = _engine(c, data, None)
    live.append(single)
    cap, layout = c.capacity, c.layout(0)
    ins = [_inputs(c, 0, l) for l in range(c.layers)]
    outs = [[torch.empty_like(x) for x in xs] for xs, _ in ins]

    def step():
        for l, (xs, rins) in enumerate(ins):
            lb.layer(l, xs, rins, outs[l], layout, cap)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    torch.cuda.synchronize()
    for i in range(3):
        for l, (xs, _) in enumerate(ins):
            for r, x in enumerate(xs):
                x.copy_(X.make_x(x.shape[0], c.H, x.dtype, seed=31 * i + 7 * l + r + 1, dev="cuda"))
        g.replay()
        torch.cuda.synchronize()
        got = [[o.clone() for o in ol] for ol in outs]
        step()
        torch.cuda.synchronize()
        for l, (xs, rins) in enumerate(ins):
            for r, x in enumerate(xs):
                _same(got[l][r], outs[l][r], f"replay {i} layer {l} rank {r}: graph vs eager")
                _same(got[l][r], _single(c, single, l, x, rins[r]).reshape(x.shape), f"replay {i} layer {l} rank {r}: graph vs single")
    del g
    _release(live)


def test_refusals(lib_built, live):
    """The inline layout past 4E = 2H is refused without a launch and the context then runs a correct step in the separate
    layout; a context with fp32 numerics is refused by the exchange."""
    from moe_infinity_b200 import _lib as L
    _release(live)
    wide = EP.EpCase("e256_h256", EP.GREEDY, 256, 512, 256, 8, "bf16", 2, ((16, 16),), (EP.SEPARATE,),
                     "inline counts past 4E = 2H", design=EP.BY_NAME["e256_n2_el128"].design)
    data = _data(wide)
    lb = EP.LoopbackEP(wide, lambda r: _engine(wide, data, r))
    live.append(lb)
    single = _engine(wide, data, None)
    live.append(single)
    xs, rins = _inputs(wide, 0, 0)
    lb.engines[0].route(0, xs[0], scores=rins[0][1])
    b = lb.buffers(EP.INLINE, wide.capacity)
    with pytest.raises(L.B2MError):
        lb.ops[0].pack(2, 0, wide.capacity, 16, b["send"][0])
    run_row(wide, lb, single, data)

    small = EP.EpCase("fp32num", EP.MIXTRAL, 256, 512, 8, 2, "bf16", 2, ((4, 4),), (EP.INLINE,), "fp32 numerics",
                      design=EP._d_uneven)
    sdata = _data(small)
    eng = _engine(small, sdata, 0, numerics=L.NUMERICS_FP32)
    live.append(eng)
    xs, rins = _inputs(small, 0, 0)
    eng.route(0, xs[0], router_logits=rins[0][0])
    from moe_infinity_b200.ep import _EngineOps
    send = torch.zeros(2, small.capacity + 1, small.H, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(L.B2MError) as ei:
        _EngineOps(eng).pack(2, 0, small.capacity, 4, send)
    assert ei.value.code == L.B2M_EUNSUPPORTED and "fp32" in str(ei.value)
    _release(live)
