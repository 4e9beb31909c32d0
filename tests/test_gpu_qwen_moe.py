"""GPU: Qwen2-MoE / Qwen3-MoE layers (router=ROUTER_QWEN_MOE) against tests/qwen_moe_oracle.py and the transformers
models.

* routing, T = 1..1024 through both routing paths (small-T and large-T kernels), fused gate and logits input, norm on and
  off: indices and weights equal the oracle's on the kernel's own logits and probabilities;
* the combine: torch.equal to the oracle's chain fed the engine's own topk_idx / topk_w, expert outputs, shared-expert
  output and gate values; each gate value torch's sigmoid of torch's F.linear(x, g) or of a logit one model-dtype ulp
  from it (the dot's fp32 summation order);
* the fixtures written from the literal HF blocks, full-size layers at published shapes, fp8 / int4 engines against
  engines holding the dequantised weights, offload and captured decode, and patched transformers models."""
from __future__ import annotations

import copy
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_golden_qwen_moe as G  # noqa: E402
import qwen_moe_oracle as Q  # noqa: E402

pytestmark = pytest.mark.gpu


def _weights(E, H, I, SI, dtype, seed, gate_std=0.5, sg_std=0.5):
    g = torch.Generator().manual_seed(seed)
    w = dict(gate_w=(torch.randn(E, H, generator=g) * gate_std / H ** 0.5 * 8),
             gate_up=torch.randn(E, 2 * I, H, generator=g) * (1.5 / H ** 0.5),
             down=torch.randn(E, H, I, generator=g) * (1.5 / I ** 0.5))
    if SI:
        w["shared"] = [torch.randn(SI, H, generator=g) * (1.5 / H ** 0.5), torch.randn(SI, H, generator=g) * (1.5 / H ** 0.5),
                       torch.randn(H, SI, generator=g) * (1.5 / SI ** 0.5)]
        w["shared_gate_w"] = torch.randn(1, H, generator=g) * (sg_std * 8 / H ** 0.5)
    out = {}
    for key, v in w.items():
        out[key] = [t.to(dtype).cuda() for t in v] if isinstance(v, list) else v.to(dtype).cuda()
    return out


def _engine(w, E, k, H, I, SI, dtype, norm, max_tokens=1024, L_=1, num_slots=0, resident=True, expert_dtype=None, **kw):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200.hf import _load
    eng = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                    router=L.ROUTER_QWEN_MOE, norm_topk_prob=norm, shared_inter=SI, max_tokens=max_tokens,
                    num_slots=num_slots or L_ * E, expert_dtype=expert_dtype, **kw)
    for l in range(L_):
        for e in range(E):
            _load(eng, l, e, [w["gate_up"][e, :I], w["gate_up"][e, I:], w["down"][e]], resident)
        if SI:
            eng.register_shared(l, w["shared"])
            eng.set_shared_gate(l, w["shared_gate_w"])
        eng.set_gate(l, w["gate_w"])
    return eng


def _ulp(t: torch.Tensor) -> torch.Tensor:
    a = t.float().abs()
    return torch.nextafter(t.abs(), torch.full_like(t, float("inf"))).float() - a


def _replay_combine(eng, T, SI):
    """The oracle's combine chain on the engine's own workspace tensors."""
    idx, w, row_of = eng.ws("topk_idx", T).long(), eng.ws("topk_w", T), eng.ws("row_of", T).long()
    y = eng.ws("y", T)[row_of.clamp(min=0)]                                          # [T,k,H] fp32
    s = eng.ws("y_shared", T) if SI else None
    g = eng.ws("shared_gate", T) if SI else None
    return Q.qwen_combine(y, torch.where(row_of < 0, -1, idx), w, eng.dtype, s, g)


def _equal_or_splitk(a, b, what="", ea=None, eb=None, T=0, SI=0):
    """Equal, or -- the down projection's split-K fp32 atomics add in a run-dependent order, so an expert output can differ
    in its last fp32 bit even between two calls of one engine -- a few elements apart.  With the engines given, each output
    must then equal the combine chain replayed on that engine's own inputs, and the fp32 expert outputs must agree to
    summation order: the difference comes from the GEMMs' atomics only."""
    if torch.equal(a, b):
        return
    bad = a != b
    assert bad.float().mean() <= 1e-3, (what, int(bad.sum()))
    if ea is not None:
        assert torch.equal(a, _replay_combine(ea, T, SI)) and torch.equal(b, _replay_combine(eb, T, SI)), what
        ya, yb = ea.ws("y", T), eb.ws("y", T)
        assert torch.allclose(ya, yb, rtol=1e-5, atol=1e-5 * yb.abs().max().item()), what
    else:
        diff = (a.float() - b.float()).abs()
        assert bool((diff[bad] <= 4 * _ulp(b)[bad] + 2 * _ulp(b.abs().amax(dim=-1, keepdim=True).expand_as(b))[bad]).all()), \
            (what, int(bad.sum()), diff.max().item())


# ---------------------------------------------------------------- routing sweep
@pytest.mark.parametrize("E,k", [(60, 4), (128, 8)])
@pytest.mark.parametrize("norm", [False, True])
def test_routing_sweep_matches_oracle(lib_built, E, k, norm):
    H, I, dtype = 256, 128, torch.bfloat16
    w = _weights(E, H, I, 0, dtype, seed=E + k + norm)
    eng = _engine(w, E, k, H, I, 0, dtype, norm)
    g = torch.Generator().manual_seed(5)
    for T in (1, 2, 7, 33, 100, 256, 257, 600, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        for kind in ("fused", "logits"):
            if kind == "fused":
                eng.route(0, x)
            else:
                eng.route(0, x, router_logits=F.linear(x, w["gate_w"]))
            torch.cuda.synchronize()
            lg = eng.ws("logits", T)
            assert lg.dtype == dtype
            if kind == "logits":
                assert torch.equal(lg, F.linear(x, w["gate_w"])), T
            else:   # the fused gate: the fp64 dot rounded to the model dtype, up to fp32 summation order
                exact = x.double() @ w["gate_w"].double().t()
                eps = torch.finfo(dtype).eps
                assert bool(((lg.double() - exact).abs() <= eps * exact.abs() + 1e-4).all()), T
            p = eng.ws("scores", T)
            assert torch.allclose(p, torch.softmax(lg.float(), dim=-1), rtol=2e-5, atol=1e-8)
            ridx, rw = Q.qwen_route_from_probs(p, k, norm)
            assert torch.equal(eng.ws("topk_idx", T).long(), ridx), (T, kind)
            assert torch.equal(eng.ws("topk_w", T), rw), (T, kind)
            tied = Q.topk_ties(lg, k)
            oidx, _ = Q.qwen_route(lg, k, norm)
            assert torch.equal(oidx[~tied].sort(-1).values, ridx[~tied].sort(-1).values), (T, kind)
    assert eng.stats()["host_syncs"] == 0


# ---------------------------------------------------------------- combine chain on the engine's own inputs
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("SI", [0, 384])
def test_combine_replays_oracle_chain(lib_built, dtype, SI):
    E, k, H, I = 60, 4, 384, 256
    w = _weights(E, H, I, SI, dtype, seed=11, sg_std=8.0)
    eng = _engine(w, E, k, H, I, SI, dtype, norm=False)
    g = torch.Generator().manual_seed(6)
    seen = set()
    for T in (1, 5, 64, 300, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        out = eng.forward(0, x, router_logits=F.linear(x, w["gate_w"]))
        torch.cuda.synchronize()
        assert torch.equal(out, _replay_combine(eng, T, SI)), T
        if SI:
            # the engine's logit is torch's up to the dot's fp32 summation order: one model-dtype ulp either way; the gate
            # value is then exactly torch's sigmoid of one of those three logits
            gv, lg = eng.ws("shared_gate", T), F.linear(x, w["shared_gate_w"]).reshape(-1)
            cands = [torch.sigmoid(torch.nextafter(lg, torch.full_like(lg, v))) for v in (-float("inf"), float("inf"))]
            assert bool(((gv == torch.sigmoid(lg)) | (gv == cands[0]) | (gv == cands[1])).all()), T
            assert (gv == torch.sigmoid(lg)).float().mean() > 0.95, T
            seen |= {v for v in (0.0, 1.0) if bool((gv == v).any())}
    assert not SI or seen == {0.0, 1.0}, f"gate values reached only {seen} of 0 and 1"


# ---------------------------------------------------------------- fixtures from the literal HF blocks
@pytest.mark.parametrize("name", list(G.CASES))
def test_engine_reproduces_fixtures(lib_built, name):
    from test_gpu_parity import hidden_close
    d = G.load(name)
    SI, E, k, H, I = d["shared_I"], d["E"], d["k"], d["H"], d["I"]
    w = {key: ([t.cuda() for t in v] if isinstance(v, list) else v.cuda()) for key, v in d.items()
         if key in ("gate_w", "gate_up", "down", "shared", "shared_gate_w")}
    eng = _engine(w, E, k, H, I, SI, torch.bfloat16, d["norm_topk_prob"], max_tokens=64)
    x = d["x"].cuda()
    out = eng.forward(0, x, router_logits=d["logits"].cuda())
    torch.cuda.synchronize()
    tied = Q.topk_ties(d["logits"], k)
    idx, wt = eng.ws("topk_idx", x.shape[0]).long().cpu(), eng.ws("topk_w", x.shape[0]).cpu()
    assert torch.equal(idx[~tied].sort(-1).values, d["topk_idx"][~tied].sort(-1).values)
    # weights by expert: HF's softmax ran on the CPU (another exp and summation order): equal to rtol 2e-5
    o1, o2 = idx.argsort(-1), d["topk_idx"].argsort(-1)
    assert torch.allclose(wt.gather(1, o1)[~tied], d["topk_w"].gather(1, o2)[~tied], rtol=2e-5, atol=0)
    if k == 1:
        assert torch.equal(wt, torch.ones_like(wt))
    hidden_close(out[~tied.cuda()], d["out"][~tied], None, torch.bfloat16, name)


# ---------------------------------------------------------------- full-size layers at published shapes
SHAPES = {
    # name: (E, k, H, I, shared I, norm_topk_prob)
    "qwen1.5-moe-a2.7b": (60, 4, 2048, 1408, 5632, False),
    "qwen2-57b-a14b": (64, 8, 3584, 2560, 20480, False),
    "qwen3-30b-a3b": (128, 8, 2048, 768, 0, True),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fullsize_layer_matches_torch(lib_built, shape):
    from test_gpu_parity import hidden_close
    E, k, H, I, SI, norm = SHAPES[shape]
    dtype = torch.bfloat16
    w = _weights(E, H, I, SI, dtype, seed=21, sg_std=1.0)
    eng = _engine(w, E, k, H, I, SI, dtype, norm)
    g = torch.Generator().manual_seed(7)
    for T in (1, 8, 64, 333, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        lg = F.linear(x, w["gate_w"])
        out = eng.forward(0, x, router_logits=lg)
        ref, _, ridx, _ = Q.qwen_block(x, w["gate_w"], w["gate_up"], w["down"], k, norm, w.get("shared"),
                                       w.get("shared_gate_w"))
        torch.cuda.synchronize()
        assert torch.equal(out, _replay_combine(eng, T, SI)), (shape, T)
        assert torch.equal(eng.ws("topk_idx", T).long().sort(-1).values, ridx.sort(-1).values), (shape, T)
        hidden_close(out, ref.cpu(), None, dtype, f"{shape} T={T}")
    del eng
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- weight formats
@pytest.mark.parametrize("fmt", ["fp8", "int4_bf16", "int4_f16"])
def test_format_engines_equal_dequantised(lib_built, fmt):
    from moe_infinity_b200 import fp8 as F8
    from moe_infinity_b200 import int4 as I4
    E, k, H, I, SI = 60, 4, 2048, 1408, 5632
    dtype = torch.float16 if fmt == "int4_f16" else torch.bfloat16
    w = _weights(E, H, I, SI, dtype, seed=31, sg_std=1.0)
    # the weights a dtype engine must hold to compute what the quantised engine computes
    deq = dict(w)
    gu, dn = w["gate_up"].clone(), w["down"].clone()
    for e in range(E):
        mats = [w["gate_up"][e, :I], w["gate_up"][e, I:], w["down"][e]]
        if fmt == "fp8":
            mats = [F8.dequantize_block128(*F8.quantize_block128(m), dtype) for m in mats]
        else:
            mats = [I4.dequantize_g128(*I4.quantize_g128(m, scale_dtype=dtype), dtype) for m in mats]
        gu[e, :I], gu[e, I:], dn[e] = mats
    deq["gate_up"], deq["down"] = gu, dn
    q = _engine(w, E, k, H, I, SI, dtype, False, expert_dtype=torch.float8_e4m3fn if fmt == "fp8" else torch.uint4)
    ref = _engine(deq, E, k, H, I, SI, dtype, False)
    g = torch.Generator().manual_seed(8)
    for T in (1, 16, 200, 1024):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        lg = F.linear(x, w["gate_w"])
        a = q.forward(0, x, router_logits=lg)
        b = ref.forward(0, x, router_logits=lg)
        torch.cuda.synchronize()
        _equal_or_splitk(a, b, f"{fmt} T={T}", q, ref, T, SI)


# ---------------------------------------------------------------- offload and captured decode
def test_offload_equals_resident_and_graph_equals_eager(lib_built):
    from moe_infinity_b200 import DecodeSession
    E, k, H, I, SI, L_ = 60, 4, 2048, 1408, 5632, 2
    dtype = torch.bfloat16
    w = _weights(E, H, I, SI, dtype, seed=41, sg_std=1.0)
    res = _engine(w, E, k, H, I, SI, dtype, False, L_=L_)
    off = _engine(w, E, k, H, I, SI, dtype, False, L_=L_, num_slots=40, resident=False)
    g = torch.Generator().manual_seed(9)
    for T in (1, 8, 64):
        x = torch.randn(T, H, generator=g).to(dtype).cuda()
        for l in range(L_):
            a = res.forward(l, x)
            b = off.forward(l, x)
            torch.cuda.synchronize()
            _equal_or_splitk(a, b, f"offload l={l} T={T}", res, off, T, SI)
    T = 8
    sess = DecodeSession(res, T)
    xs = torch.randn(L_, T, H, generator=g).to(dtype)
    sess.x_host.copy_(xs)
    eager = sess.step().clone()
    sess.capture()
    for it in range(3):
        sess.x_host.copy_(xs)
        _equal_or_splitk(sess.step(), eager, f"graph replay {it}")
    # the captured graph reads the shared gate's contents at replay
    res._shared_gates[0].mul_(-1.0)
    sess.x_host.copy_(xs)
    flipped = sess.step().clone()
    assert not torch.equal(flipped[0], eager[0])
    assert res.stats()["host_syncs"] == 0


# ---------------------------------------------------------------- transformers models
def _tiny(kind):
    if kind == "qwen2":
        from transformers import Qwen2MoeConfig as C_, Qwen2MoeForCausalLM as M_
        cfg = C_(vocab_size=512, hidden_size=256, intermediate_size=512, moe_intermediate_size=128,
                 shared_expert_intermediate_size=384, num_hidden_layers=3, num_attention_heads=4, num_key_value_heads=2,
                 num_experts=16, num_experts_per_tok=4, norm_topk_prob=False, mlp_only_layers=[0],
                 max_position_embeddings=128)
    else:
        from transformers import Qwen3MoeConfig as C_, Qwen3MoeForCausalLM as M_
        cfg = C_(vocab_size=512, hidden_size=256, intermediate_size=512, moe_intermediate_size=128, num_hidden_layers=2,
                 num_attention_heads=4, num_key_value_heads=2, head_dim=64, num_experts=32, num_experts_per_tok=8,
                 norm_topk_prob=True, max_position_embeddings=128)
    torch.manual_seed(0)
    model = M_(cfg).to(torch.bfloat16).cuda().eval()
    with torch.no_grad():      # HF's tiny init (std 0.02) gives near-uniform routing; spread the router and the gate
        for layer in model.model.layers:
            if hasattr(layer.mlp, "gate") and hasattr(layer.mlp, "experts"):
                layer.mlp.gate.weight.mul_(20.0)
                if hasattr(layer.mlp, "shared_expert_gate"):
                    layer.mlp.shared_expert_gate.weight.mul_(50.0)
    return model


@pytest.mark.parametrize("kind", ["qwen2", "qwen3"])
def test_patched_qwen_matches_hf(lib_built, kind):
    from moe_infinity_b200.hf import B200QwenMoeAdapter, patch_qwen_moe
    ref = _tiny(kind)
    ours = copy.deepcopy(ref)
    eng = patch_qwen_moe(ours, max_tokens=256)
    adapters = [type(layer.mlp) is B200QwenMoeAdapter for layer in ours.model.layers]
    assert adapters == ([False, True, True] if kind == "qwen2" else [True, True])
    ids = torch.randint(0, 512, (2, 24), device="cuda")
    with torch.no_grad():
        a = ref(ids).logits.float()
        b = ours(ids).logits.float()
    rms = a.pow(2).mean().sqrt()
    err = (a - b).abs()
    assert err.max() <= 0.08 * rms and err.pow(2).mean().sqrt() <= 0.01 * rms, (err.max().item(), rms.item())
    assert (a.argmax(-1) == b.argmax(-1)).float().mean() > 0.97
    with torch.no_grad():
        ga = ref.generate(ids[:, :8], max_new_tokens=8, do_sample=False)
        gb = ours.generate(ids[:, :8], max_new_tokens=8, do_sample=False)
    assert (ga == gb).float().mean() > 0.9
    assert eng.stats()["kernel_launches"] > 0 and eng.stats()["host_syncs"] == 0
