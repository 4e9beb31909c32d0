"""GPU: the grouped expert GEMMs (csrc/grouped_gemm.cu K3 / K4, and the CUDA-core paths) compute exactly the float64
reference on every row of tests/gemm_exact_cases.py -- torch.equal, no tolerance.

The rows' data keep every partial sum an integer number of units below 2^22 (see gemm_exact_cases.py), so the right answer
is exact in fp32 whatever the split-K / stream-K grouping and the order of the fp32 atomics.  Per row:
* one shipped forward (router logits or scores designed for the row's per-expert token counts; Switch / NLLB rows route
  from a mask): ws("hmid") and ws("y") equal the reference row by row, DeepSeek's ws("y_shared") too, and the layer output
  equals the oracle's combine replayed on those outputs with the engine's own topk_idx / topk_w;
* with every expert resident: the down projection alone (phases=2) on dense small integers written into ws("hmid");
* rows reading the 12-bit packed copy forward twice first and check that the copy was allocated.
tests/test_gemm_exact_plans.py checks on the CPU which launch plan each row runs (stated for 132 SMs)."""
from __future__ import annotations

import pytest
import torch

import gemm_exact_cases as X

pytestmark = pytest.mark.gpu

_cur = {"key": None}


def _engine_for(c: X.Case):
    """One engine (and its experts) per engine key, kept while consecutive rows share it."""
    if _cur["key"] == c.engine_key:
        return _cur
    if _cur.get("eng") is not None:
        _cur["eng"].close()
    _cur.clear()
    _cur["key"] = None
    torch.cuda.empty_cache()
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    dt = X.DTYPES[c.dtype]
    max_t = max(r.T for r in X.CASES if r.engine_key == c.engine_key)
    eng = MoEEngine(num_layers=1, num_experts=c.E, hidden=c.H, inter=c.I, top_k=c.k, dtype=dt, expert_type=X.ETYPE[c.etype],
                    router=L.ROUTER_DEEPSEEK_GREEDY if c.etype == X.DEEPSEEK else L.ROUTER_MIXTRAL,
                    numerics=L.NUMERICS_FP32 if c.numerics == "fp32" else L.NUMERICS_REFERENCE, max_tokens=max(max_t, 16),
                    num_slots=c.slots, shared_inter=c.shared, gemm_impl=c.gemm_impl, pack_weights=c.fmt == "pk12",
                    expert_dtype={"fp8": torch.float8_e4m3fn, "int4": torch.uint4}.get(c.fmt))
    experts = []
    for e in range(c.E):
        ex = X.make_expert(c, seed=1000 + e, dev="cuda")
        if c.slots:
            eng.register_expert(0, e, ex.load, scales=ex.scales, zeros=ex.zeros)
        else:
            eng.load_expert(0, e, ex.load, scales=ex.scales, zeros=ex.zeros)
        experts.append(ex)
    shared = None
    if c.shared:
        sc = X.Case("shared", X.DEEPSEEK, c.H, c.shared, 1, 1, c.dtype, "bf16", c.T, (c.T,), c.plan)
        shared = (sc, X.make_expert(sc, seed=999, dev="cuda"))
        eng.register_shared(0, shared[1].w)
    torch.cuda.synchronize()
    _cur.update(key=c.engine_key, eng=eng, experts=experts, shared=shared, free0=torch.cuda.mem_get_info()[0])
    return _cur


def _same(got: torch.Tensor, want: torch.Tensor, what: str):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if torch.equal(got, want):
        return
    bad = (got != want).nonzero()
    r, col = bad[0].tolist()
    raise AssertionError(f"{what}: {bad.shape[0]} of {got.numel()} elements differ; first at row {r} col {col}: "
                         f"got {got[r, col].item()} want {want[r, col].item()}; rows hit {bad[:, 0].unique().numel()}, "
                         f"cols hit {bad[:, 1].unique().numel()}")


def _route_and_run(c: X.Case, eng, x):
    if c.routed_by_forward:
        lg = X.router_logits(c.counts, c.T, c.k).cuda()
        if c.etype == X.DEEPSEEK:
            return eng.forward(0, x, scores=torch.softmax(lg, dim=-1))
        return eng.forward(0, x, router_logits=lg)
    eng.route_from_mask(0, x, X.route_mask(c.counts, c.T, c.k).cuda())
    eng.run_experts(0, c.T)
    return None


def _replay_combine(c: X.Case, eng, y: torch.Tensor, y_shared):
    """oracle mixtral_block / deepseek_block combine: experts in ascending id, every op in the model dtype (DeepSeek: the
    product with the fp32 weight in fp32, the add rounded), then + the shared expert's output."""
    dt = X.DTYPES[c.dtype]
    T = c.T
    idx, w, row_of = eng.ws("topk_idx", T).long(), eng.ws("topk_w", T), eng.ws("row_of", T).long()
    order = idx.argsort(dim=1)
    final = torch.zeros(T, c.H, dtype=dt, device="cuda")
    for j in range(c.k):
        col = order[:, j:j + 1]
        yj = y[row_of.gather(1, col).squeeze(1)].to(dt)
        wj = w.gather(1, col)
        if c.etype == X.MIXTRAL:
            final = final + yj * wj.to(dt)
        else:
            final = (final.float() + yj.float() * wj).to(dt)
    if y_shared is not None:
        final = final + y_shared.to(dt)
    return final


@pytest.mark.parametrize("name", [c.name for c in X.CASES])
def test_expert_gemms_are_exact(lib_built, name):
    c = X.BY_NAME[name]
    st = _engine_for(c)
    eng, experts = st["eng"], st["experts"]
    dt = X.DTYPES[c.dtype]
    x = X.make_x(c.T, c.H, dt, seed=c.T, dev="cuda")
    if c.fmt == "pk12":
        _route_and_run(c, eng, x)          # the second eager forward after the load packs the slots
        _route_and_run(c, eng, x)
        torch.cuda.synchronize()
        if (c.H, c.I) == (X.MH, X.MI):
            assert st["free0"] - torch.cuda.mem_get_info()[0] > 1.5e9, "the packed copy was not allocated"
    out = _route_and_run(c, eng, x)
    torch.cuda.synchronize()
    T, k = c.T, c.k
    assert eng.ws("counts", T).tolist() == list(c.counts), "routing did not produce the designed counts"
    offs = eng.ws("offsets", T).tolist()
    perm = eng.ws("perm_token", T).long()
    want_rows = X.expert_rows(c.counts, T, k)
    hmid, y = eng.ws("hmid", T), eng.ws("y", T)
    y_all = torch.empty(T * k, c.H, dtype=torch.float32, device="cuda")
    for e in range(c.E):
        r0, r1 = offs[e], offs[e + 1]
        if r0 == r1:
            continue
        tok = perm[r0:r1]
        assert torch.equal(tok.cpu(), want_rows[e]), f"expert {e}: rows hold other tokens"
        h_ref, y_ref = X.reference(c, x[tok], experts[e].w)
        _same(hmid[r0:r1], h_ref, f"{name} expert {e} hmid")
        _same(y[r0:r1], y_ref, f"{name} expert {e} y")
        y_all[r0:r1] = y_ref
    y_shared = None
    if c.shared:
        sc, sx = st["shared"]
        y_shared = X.reference(sc, x, sx.w)[1]
        _same(eng.ws("y_shared", T), y_shared, f"{name} y_shared")
    if out is not None and c.numerics == "reference" and c.dtype != "f32":
        _same(out.reshape(T, c.H), _replay_combine(c, eng, y_all, y_shared), f"{name} layer output")

    if c.slots == 0:
        # the down projection alone, on dense data (reuses the slot row the forward above left: every expert resident)
        h2 = X.make_hmid(T * k, c.I, dt, seed=7 + T, dev="cuda")
        hmid.copy_(h2)
        y.zero_()
        eng.run_experts(0, T, phases=2)
        torch.cuda.synchronize()
        for e in range(c.E):
            r0, r1 = offs[e], offs[e + 1]
            if r0 < r1:
                _same(y[r0:r1], X.reference(c, None, experts[e].w, hmid=h2[r0:r1])[1], f"{name} expert {e} y (dense hmid)")


def test_release_engine(lib_built):
    if _cur.get("eng") is not None:
        _cur["eng"].close()
    _cur.clear()
    _cur["key"] = None
    torch.cuda.empty_cache()
