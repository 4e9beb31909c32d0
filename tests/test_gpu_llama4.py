"""GPU: Llama 4 MoE layers (router=ROUTER_LLAMA4) against tests/llama4_oracle.py and the transformers model.

* routing, T = 1..1024 through both routing paths (small-T and large-T kernels), E in {16, 128}, k in {1, 2, 8}, bf16 and
  f16, fused gate and logits input: indices and weights equal the oracle's on the logits the kernel used, the scores are
  the sigmoid of every logit, and every gathered row is round(x[t] * w);
* the combine: torch.equal to the oracle's chain fed the engine's own expert and shared-expert outputs, both numerics;
* the fixtures written from the literal HF block, a Scout-shaped and a Maverick-shaped layer against a torch restatement,
  fp8 / int4 engines against engines holding the dequantised weights, offload, captured decode, the look-ahead
  prediction and a patched transformers model with interleaved dense layers."""
from __future__ import annotations

import copy
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import llama4_oracle as O  # noqa: E402
import make_golden_llama4 as G  # noqa: E402

pytestmark = pytest.mark.gpu


def _expert(seed, e, H, I, dtype):
    """Expert e's (gate [I,H], up [I,H], down [H,I]) from its own seed, generated on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed * 1000 + e)
    return [(torch.randn(I, H, generator=g, device="cuda") * (1.5 / H ** 0.5)).to(dtype),
            (torch.randn(I, H, generator=g, device="cuda") * (1.5 / H ** 0.5)).to(dtype),
            (torch.randn(H, I, generator=g, device="cuda") * (1.5 / I ** 0.5)).to(dtype)]


def _router(seed, E, H, dtype, std=4.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(E, H, generator=g, device="cuda") * (std / H ** 0.5)).to(dtype)


def _engine(E, k, H, I, dtype, seed, max_tokens=1024, L_=1, num_slots=0, resident=True, expert_dtype=None,
            experts=None, shared=None, **kw):
    """A Llama 4 engine whose layer l holds the experts of seed + l (or `experts[e]`, mats in the model dtype), the shared
    expert of seed key E (or `shared`) and the router of seed + l."""
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200.hf import _load
    eng = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                    router=L.ROUTER_LLAMA4, shared_inter=I, max_tokens=max_tokens, num_slots=num_slots or L_ * E,
                    expert_dtype=expert_dtype, **kw)
    for l in range(L_):
        for e in range(E):
            _load(eng, l, e, experts[e] if experts is not None else _expert(seed + l, e, H, I, dtype), resident)
        eng.register_shared(l, shared if shared is not None else _expert(seed + l, E, H, I, dtype))
        eng.set_gate(l, _router(seed + l, E, H, dtype))
    return eng


def _replay_combine(eng, T, fp32=False):
    """The oracle's combine chain on the engine's own workspace tensors."""
    idx, row_of = eng.ws("topk_idx", T).long(), eng.ws("row_of", T).long()
    y = eng.ws("y", T)[row_of.clamp(min=0)]                                          # [T,k,H] fp32
    return O.llama4_combine(y, torch.where(row_of < 0, -1, idx), eng.dtype, eng.ws("y_shared", T), fp32)


def _restate(x, logits, seed, k, H, I, dtype, experts=None):
    """Torch restatement of the layer: the oracle's routing, then each chosen expert's SwiGLU (F.linear, every op in the
    model dtype) on its scaled input rows, then the oracle's combine."""
    idx, w = O.llama4_route(logits, k)
    xs = O.scaled_inputs(x, w)                                                       # [T,k,H]
    y = torch.zeros(x.shape[0], k, H, dtype=dtype, device=x.device)
    for e in idx.unique().tolist():
        gw, uw, dw = experts[e] if experts is not None else _expert(seed, e, H, I, dtype)
        sel = idx == e
        y[sel] = O.shared_expert(xs[sel], gw, uw, dw)
    s = O.shared_expert(x, *_expert(seed, logits.shape[1], H, I, dtype))
    return O.llama4_combine(y, idx, dtype, s), idx


def _equal_or_splitk(a, b, what, ea=None, eb=None, T=0):
    """Equal, or -- the down projection's split-K fp32 atomics add in a run-dependent order, so an expert output can differ
    in its last fp32 bit between two calls -- a few elements apart, each engine's output then equal to the combine chain
    replayed on its own inputs and the fp32 expert outputs equal up to summation order."""
    if torch.equal(a, b):
        return
    bad = a != b
    assert bad.float().mean() <= 1e-3, (what, int(bad.sum()))
    if ea is not None:
        assert torch.equal(a, _replay_combine(ea, T)) and torch.equal(b, _replay_combine(eb, T)), what
        ya, yb = ea.ws("y", T), eb.ws("y", T)
        assert torch.allclose(ya, yb, rtol=1e-5, atol=1e-5 * yb.abs().max().item()), what
    else:
        ulp = torch.nextafter(b.abs(), torch.full_like(b, float("inf"))).float() - b.float().abs()
        big = ulp.amax(dim=-1, keepdim=True).expand_as(b)
        assert bool(((a.float() - b.float()).abs()[bad] <= 4 * ulp[bad] + 2 * big[bad]).all()), what


# ---------------------------------------------------------------- routing sweep
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("E,k", [(16, 1), (16, 2), (16, 8), (128, 1), (128, 2), (128, 8)])
def test_routing_sweep_matches_oracle(lib_built, E, k, dtype):
    H, I = 256, 128
    eng = _engine(E, k, H, I, dtype, seed=E + k)
    gw = _router(E + k, E, H, dtype)
    g = torch.Generator().manual_seed(5)
    for T in (1, 2, 7, 33, 100, 256, 257, 600, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        for kind in ("fused", "logits"):
            if kind == "fused":
                eng.route(0, x)
            else:
                eng.route(0, x, router_logits=F.linear(x, gw))
            torch.cuda.synchronize()
            lg = eng.ws("logits", T)
            assert lg.dtype == dtype
            if kind == "logits":
                assert torch.equal(lg, F.linear(x, gw)), T
            else:   # the fused gate: the fp64 dot rounded to the model dtype, up to fp32 summation order
                exact = x.double() @ gw.double().t()
                eps = torch.finfo(dtype).eps
                assert bool(((lg.double() - exact).abs() <= eps * exact.abs() + 1e-4).all()), T
            assert torch.equal(eng.ws("scores", T), torch.sigmoid(lg.float())), (T, kind)
            ridx, rw = O.llama4_route(lg, k)
            idx, w = eng.ws("topk_idx", T).long(), eng.ws("topk_w", T)
            assert torch.equal(idx, ridx), (T, kind)
            assert torch.equal(w, rw), (T, kind)
            row_of, xp = eng.ws("row_of", T).long(), eng.ws("xp", T)
            assert bool((row_of >= 0).all())
            assert torch.equal(xp[row_of], O.scaled_inputs(x, w)), (T, kind)
    assert eng.stats()["host_syncs"] == 0


# ---------------------------------------------------------------- combine chain on the engine's own inputs
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("fp32", [False, True])
def test_combine_replays_oracle_chain(lib_built, dtype, k, fp32):
    from moe_infinity_b200 import _lib as L
    E, H, I = 16, 384, 256
    eng = _engine(E, k, H, I, dtype, seed=11, numerics=L.NUMERICS_FP32 if fp32 else L.NUMERICS_REFERENCE)
    gw = _router(11, E, H, dtype)
    g = torch.Generator().manual_seed(6)
    for T in (1, 5, 64, 300, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        out = eng.forward(0, x, router_logits=F.linear(x, gw))
        torch.cuda.synchronize()
        assert torch.equal(out, _replay_combine(eng, T, fp32)), T


# ---------------------------------------------------------------- fixtures from the literal HF block
@pytest.mark.parametrize("name", list(G.CASES))
def test_engine_reproduces_fixtures(lib_built, name):
    from test_gpu_parity import hidden_close
    d = G.load(name)
    E, k, H, I = d["E"], d["k"], d["H"], d["I"]
    dtype = G.DTYPES[d["dtype"]]
    gu, dn = d["gate_up"].cuda(), d["down"].cuda()
    experts = [[gu[e][:, :I].t().contiguous(), gu[e][:, I:].t().contiguous(), dn[e].t().contiguous()] for e in range(E)]
    eng = _engine(E, k, H, I, dtype, seed=0, max_tokens=64, experts=experts, shared=[t.cuda() for t in d["shared"]])
    x = d["x"].cuda()
    out = eng.forward(0, x, router_logits=d["logits"].cuda())
    torch.cuda.synchronize()
    T = x.shape[0]
    assert torch.equal(eng.ws("topk_idx", T).long().cpu(), d["topk_idx"])
    assert torch.equal(eng.ws("topk_w", T).cpu(), d["topk_w"])
    hidden_close(out, d["out"], None, dtype, name)


# ---------------------------------------------------------------- full-size layers at published shapes
SHAPES = {
    # name: (E, k, H, I)
    "llama4-scout-17b-16e": (16, 1, 5120, 8192),
    "llama4-maverick-17b-128e": (128, 1, 5120, 8192),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fullsize_layer_matches_torch(lib_built, shape):
    from test_gpu_parity import hidden_close
    E, k, H, I = SHAPES[shape]
    dtype = torch.bfloat16
    eng = _engine(E, k, H, I, dtype, seed=21)
    gw = _router(21, E, H, dtype)
    g = torch.Generator().manual_seed(7)
    for T in (1, 8, 64, 333, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        lg = F.linear(x, gw)
        out = eng.forward(0, x, router_logits=lg)
        torch.cuda.synchronize()
        assert torch.equal(out, _replay_combine(eng, T)), (shape, T)
        ref, ridx = _restate(x, lg, 21, k, H, I, dtype)
        assert torch.equal(eng.ws("topk_idx", T).long(), ridx), (shape, T)
        hidden_close(out, ref.cpu(), None, dtype, f"{shape} T={T}")
    eng.close()
    del eng
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- weight formats
@pytest.mark.parametrize("fmt", ["fp8", "int4_bf16", "int4_f16"])
def test_format_engines_equal_dequantised(lib_built, fmt):
    from moe_infinity_b200 import fp8 as F8
    from moe_infinity_b200 import int4 as I4
    E, k, H, I = 16, 1, 2048, 4096
    dtype = torch.float16 if fmt == "int4_f16" else torch.bfloat16
    raw = [_expert(31, e, H, I, dtype) for e in range(E)]
    if fmt == "fp8":
        deq = [[F8.dequantize_block128(*F8.quantize_block128(m), dtype) for m in mats] for mats in raw]
    else:
        deq = [[I4.dequantize_g128(*I4.quantize_g128(m, scale_dtype=dtype), dtype) for m in mats] for mats in raw]
    q = _engine(E, k, H, I, dtype, seed=31, experts=raw,
                expert_dtype=torch.float8_e4m3fn if fmt == "fp8" else torch.uint4)
    ref = _engine(E, k, H, I, dtype, seed=31, experts=deq)
    gw = _router(31, E, H, dtype)
    g = torch.Generator().manual_seed(8)
    for T in (1, 16, 200, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        lg = F.linear(x, gw)
        a = q.forward(0, x, router_logits=lg)
        b = ref.forward(0, x, router_logits=lg)
        torch.cuda.synchronize()
        _equal_or_splitk(a, b, f"{fmt} T={T}", q, ref, T)


# ---------------------------------------------------------------- offload, captured decode, look-ahead
def test_offload_equals_resident_and_graph_equals_eager(lib_built):
    from moe_infinity_b200 import DecodeSession
    E, k, H, I, L_ = 16, 1, 2048, 4096, 2
    dtype = torch.bfloat16
    res = _engine(E, k, H, I, dtype, seed=41, L_=L_)
    off = _engine(E, k, H, I, dtype, seed=41, L_=L_, num_slots=12, resident=False)
    g = torch.Generator().manual_seed(9)
    for T in (1, 8, 64):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        for l in range(L_):
            a = res.forward(l, x)
            b = off.forward(l, x)
            torch.cuda.synchronize()
            _equal_or_splitk(a, b, f"offload l={l} T={T}", res, off, T)
    T = 8
    sess = DecodeSession(res, T)
    xs = torch.randn(L_, T, H, generator=g).to(dtype)
    sess.x_host.copy_(xs)
    eager = sess.step().clone()
    sess.capture()
    for it in range(3):
        sess.x_host.copy_(xs)
        _equal_or_splitk(sess.step(), eager, f"graph replay {it}")
    assert res.stats()["host_syncs"] == 0


def test_lookahead_counts_match_oracle(lib_built):
    """Offload context with look-ahead prefetch: the prediction made during layer l is the top-k of layer l+1's model-dtype
    logits on layer l's input.  Inputs and router rows are small multiples of 1/8, so the fp32 dots are exact on both sides
    and only the rounding to bf16 remains (the same on both)."""
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    Ln, E, k, H, I, T = 3, 16, 2, 128, 128, 6
    dtype = torch.bfloat16
    eng = MoEEngine(num_layers=Ln, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                    router=L.ROUTER_LLAMA4, shared_inter=I, max_tokens=16, num_slots=20, lookahead_prefetch=True)
    g = torch.Generator().manual_seed(11)
    for l in range(Ln):
        for e in range(E):
            eng.register_expert(l, e, [(torch.randn(I, H, generator=g) * 0.05).to(dtype),
                                       (torch.randn(I, H, generator=g) * 0.05).to(dtype),
                                       (torch.randn(H, I, generator=g) * 0.05).to(dtype)])
        eng.register_shared(l, [(torch.randn(I, H, generator=g) * 0.05).to(dtype).cuda(),
                                (torch.randn(I, H, generator=g) * 0.05).to(dtype).cuda(),
                                (torch.randn(H, I, generator=g) * 0.05).to(dtype).cuda()])
    gates = [(torch.randint(-2, 3, (E, H), generator=g).float() * 0.25).to(dtype) for _ in range(Ln)]
    for l in range(Ln):
        eng.set_gate(l, gates[l])
    for l in range(Ln - 1):
        x = (torch.randint(-2, 3, (T, H), generator=g).float() * 0.5).to(dtype)
        eng.forward(l, x.cuda())
        torch.cuda.synchronize()
        logits = (x.float() @ gates[l + 1].float().t()).to(dtype)
        idx, _ = O.llama4_route(logits, k)
        assert eng.last_lookahead() == torch.bincount(idx.flatten(), minlength=E).tolist(), l
    eng.close()


# ---------------------------------------------------------------- transformers model
def test_patched_llama4_matches_hf(lib_built):
    tr = pytest.importorskip("transformers")
    from moe_infinity_b200.hf import B200Llama4MoeAdapter, patch_llama4
    cfg = tr.Llama4TextConfig(vocab_size=512, hidden_size=256, intermediate_size=256, intermediate_size_mlp=512,
                              num_hidden_layers=4, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                              num_local_experts=16, num_experts_per_tok=1, interleave_moe_layer_step=2,
                              max_position_embeddings=128)
    torch.manual_seed(0)
    ref = tr.Llama4ForCausalLM(cfg).to(torch.bfloat16).cuda().eval()
    with torch.no_grad():      # the fused expert tensors start as zeros/empty; HF's tiny init routes near-uniformly
        for layer in ref.model.layers:
            ff = layer.feed_forward
            if hasattr(ff, "router"):
                ff.router.weight.mul_(20.0)
                ff.experts.gate_up_proj.copy_(torch.randn_like(ff.experts.gate_up_proj) * 0.02)
                ff.experts.down_proj.copy_(torch.randn_like(ff.experts.down_proj) * 0.02)
    ours = copy.deepcopy(ref)
    eng = patch_llama4(ours, max_tokens=256)
    assert [type(layer.feed_forward) is B200Llama4MoeAdapter for layer in ours.model.layers] == [False, True, False, True]
    ids = torch.randint(0, 512, (2, 24), device="cuda")
    with torch.no_grad():
        a = ref(ids).logits.float()
        b = ours(ids).logits.float()
    rms = a.pow(2).mean().sqrt()
    err = (a - b).abs()
    assert err.max() <= 0.08 * rms and err.pow(2).mean().sqrt() <= 0.01 * rms, (err.max().item(), rms.item())
    assert (a.argmax(-1) == b.argmax(-1)).float().mean() > 0.97
    assert eng.stats()["kernel_launches"] > 0 and eng.stats()["host_syncs"] == 0
