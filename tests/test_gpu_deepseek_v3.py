"""GPU: the DeepSeek-V3 router (ROUTER_DEEPSEEK_V3: sigmoid scores, per-expert correction bias, top-2-sum group selection)
in the fused routing kernels -- a sweep against the oracle over both routing paths and all router inputs, the literal
reference block and the drop-in block against the golden fixtures, a full-size layer with fp8 experts, graph capture,
the look-ahead predictor and the HuggingFace plug-in."""
import copy
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

import ref_loader  # noqa: E402
import deepseek_v3_oracle as V3  # noqa: E402
import make_golden_deepseek_v3 as GV3  # noqa: E402
from test_gpu_parity import check_permutation, hidden_close  # noqa: E402

DT = torch.bfloat16
BIAS_LEVELS = (0.0, 0.05, -0.3, -3.0)      # zero, small, negative, strongly negative (every kept choice below 0.0)


def _v3_engine(E, k, H, n_group, topk_group, norm, scale=2.5, I=128, L_=1, max_tokens=1024, **kw):
    from moe_infinity_b200 import MoEEngine, _lib as L
    kw.setdefault("num_slots", 1)
    return MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=DT, expert_type=L.EXPERT_DEEPSEEK,
                     router=L.ROUTER_DEEPSEEK_V3, n_group=n_group, topk_group=topk_group, norm_topk_prob=norm,
                     routed_scaling_factor=scale, max_tokens=max_tokens, **kw)


def _bias(E, level, g):
    if level == 0.0:
        return torch.zeros(E)
    return level + torch.randn(E, generator=g) * abs(level) * 0.5


@pytest.mark.parametrize("E,k", [(16, 4), (64, 8), (256, 8), (256, 4)])
@pytest.mark.parametrize("n_group,topk_group", [(1, 1), (4, 2), (8, 4)])
@pytest.mark.parametrize("T", [1, 31, 256, 257, 700])
def test_v3_routing_sweep(E, k, n_group, topk_group, T, lib_built):
    """Router input kinds 0 (fused fp32 gate), 1 (logits, fp32 and bf16) and 2 (sigmoid scores), norm on / off, biases from
    zero to strongly negative.  The oracle is applied to the scores the kernel saw (ws("scores")): the selection and the
    weights use the same fp32 operations in the same order, so indices and weights must be equal, ties included."""
    H = 64
    g = torch.Generator().manual_seed(E * 1009 + k * 101 + n_group * 11 + T)
    x = torch.randn(T, H, generator=g).to(DT)
    w = torch.randn(E, H, generator=g) * (2.0 / H ** 0.5)
    for norm in (False, True):
        eng = _v3_engine(E, k, H, n_group, topk_group, norm)
        eng.set_gate(0, w)
        for kind in (0, 1, 2):
            bias = _bias(E, BIAS_LEVELS[(kind + 2 * norm + T) % 4], g)
            eng.set_gate_bias(0, bias)
            logits = (torch.randn(T, E, generator=g) * 2)
            if kind == 0:
                eng.route(0, x.cuda())
            elif kind == 1:
                if T % 2:
                    logits = logits.to(DT)
                eng.route(0, x.cuda(), router_logits=logits.cuda())
            else:
                eng.route(0, x.cuda(), scores=torch.sigmoid(logits).cuda())
            torch.cuda.synchronize()
            s_gpu = eng.ws("scores", T).clone()
            if kind == 0:
                assert torch.equal(s_gpu, torch.sigmoid(eng.ws("logits", T))), "fused-gate scores != torch.sigmoid on the GPU"
            elif kind == 1:
                assert torch.equal(s_gpu, torch.sigmoid(logits.float().cuda())), "scores != torch.sigmoid on the GPU"
            else:
                assert torch.equal(s_gpu.cpu(), torch.sigmoid(logits))
            r = V3.deepseek_v3_route(s_gpu.cpu(), bias, k, n_group, topk_group, norm, 2.5, are_scores=True)
            gi, gw = eng.ws("topk_idx", T).cpu().long(), eng.ws("topk_w", T).cpu()
            assert torch.equal(gi, r.topk_idx), (norm, kind, (gi != r.topk_idx).any(-1).sum().item())
            assert torch.all((gw - r.topk_weight).abs() <= 1e-6 * r.topk_weight.abs()), (norm, kind)
        check_permutation(eng, x.cuda(), T)
        eng.close()


def _golden(name):
    import os
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".pt"), weights_only=False)
    c = GV3.build(name)
    assert torch.equal(c["hidden"], fx["hidden"]) and torch.equal(c["bias"], fx["bias"])
    return c, fx


def _golden_engine(c, **kw):
    eng = _v3_engine(c["E"], c["k"], c["H"], c["n_group"], c["topk_group"], c["norm_topk_prob"], c["routed_scaling_factor"],
                     I=c["I"], max_tokens=max(16, c["B"] * c["S"]), num_slots=c["E"],
                     shared_inter=c["I"] * c["n_shared"] if c["n_shared"] else 0, gate_dtype=torch.float32, **kw)
    for e in range(c["E"]):
        eng.load_expert(0, e, c["experts"][e])
    if c["n_shared"]:
        eng.register_shared(0, c["shared"])
    eng.set_gate(0, c["gate"].float())
    eng.set_gate_bias(0, c["bias"])
    return eng


V3_CASES = ["deepseek_v3_norm_bf16", "deepseek_v3_e64k8_bf16", "deepseek_v3_nonorm_bf16"]


@pytest.mark.parametrize("name", V3_CASES)
def test_v3_engine_matches_golden(name, lib_built):
    """The fixture's scores in (kind 2): expert indices and weights bit-exact, outputs within the V2 block bounds."""
    c, fx = _golden(name)
    eng = _golden_engine(c)
    T = c["B"] * c["S"]
    x = c["hidden"].reshape(T, -1).cuda()
    out = eng.forward(0, x, scores=fx["scores"].cuda())
    torch.cuda.synchronize()
    assert torch.equal(eng.ws("topk_idx", T).cpu().long(), fx["topk_idx"])
    assert torch.equal(eng.ws("topk_w", T).cpu(), fx["topk_weight"])
    hidden_close(out, fx["out"].reshape(T, -1), fx["out_fp32"].reshape(T, -1), DT, name)
    eng.close()


@pytest.mark.parametrize("name", V3_CASES)
def test_v3_drop_in_block_matches_golden(name, lib_built):
    """blocks.DeepseekMoEBlock with model_type "deepseek_v3": sigmoid scores in PyTorch (a GPU fp32 GEMM here, CPU in the
    fixture), the bias handed to the engine, everything else in moe_forward."""
    from moe_infinity_b200.blocks import DeepseekMoEBlock
    from moe_infinity_b200.compat import DistributedExpertExecutor
    c, fx = _golden(name)
    eng = _golden_engine(c)
    cfg = types.SimpleNamespace(model_type="deepseek_v3", num_experts_per_tok=c["k"], n_routed_experts=c["E"],
                                hidden_size=c["H"])
    blk = DeepseekMoEBlock(cfg).cuda()
    with torch.no_grad():
        blk.gate_weight.copy_(c["gate"].float())
        blk.e_score_correction_bias.copy_(c["bias"])
    ex = DistributedExpertExecutor()
    ex.set_expert_dispatcher(eng)
    blk.expert_executor, blk.layer_id = ex, 0
    with torch.no_grad():
        out = blk(c["hidden"].cuda())
    torch.cuda.synchronize()
    T = c["B"] * c["S"]
    s_gpu = eng.ws("scores", T).cpu()
    near = V3.deepseek_v3_choice_ties(s_gpu, c["bias"], c["k"], c["n_group"], c["topk_group"], rel=1e-5)
    assert near.float().mean() <= 0.2
    assert torch.equal(eng.ws("topk_idx", T).cpu().long()[~near], fx["topk_idx"][~near])
    o, r = out.reshape(T, -1)[(~near).cuda()].float().cpu(), fx["out"].reshape(T, -1)[~near].float()
    eps = torch.finfo(DT).eps
    # the weights carry the GPU gate GEMM's last fp32 bits: the V2 drop-in block's bound
    assert torch.all((o - r).abs() <= 2 * eps * r.abs() + 2 * eps * r.pow(2).mean().sqrt())
    eng.close()


needs_reference = pytest.mark.skipif(not ref_loader.available(), reason="neither /root/reference nor oracle/_ref/pyref present")


@needs_reference
@pytest.mark.parametrize("name", V3_CASES)
def test_literal_v3_block_on_gpu(name, lib_built):
    """models/deepseek.py with the literal V3 MoEGate (model_type "deepseek_v3") on the GPU over this repository's compat
    executor; the experts run in libb2m.so behind dispatch_local."""
    from moe_infinity_b200 import _lib as L
    from test_gpu_literal_blocks import _plugin
    ns = ref_loader.load()
    pytest.importorskip("moe_infinity.models.modeling_deepseek_v3", reason="the reference tree has no V3 gate module")
    c, fx = _golden(name)
    blk = ns.deepseek.DeepseekMoEBlock(GV3.config(c)).to(DT)
    blk.eval()
    with torch.no_grad():
        blk.gate.weight.copy_(c["gate"])
        blk.gate.e_score_correction_bias.copy_(c["bias"])
        if c["n_shared"] is not None:
            blk.shared_experts.gate_proj.weight.copy_(c["shared"][0])
            blk.shared_experts.up_proj.weight.copy_(c["shared"][1])
            blk.shared_experts.down_proj.weight.copy_(c["shared"][2])
    blk.gate.cuda()
    if c["n_shared"] is not None:
        blk.shared_experts.cuda()
    _, d, ex = _plugin(c, L.EXPERT_DEEPSEEK, L.DTYPE_BF16)
    blk.expert_executor, blk.layer_id = ex, 0
    with torch.no_grad():
        idx, _ = blk.gate(c["hidden"].cuda())
        out = blk(c["hidden"].cuda())
    torch.cuda.synchronize()
    T = c["B"] * c["S"]
    same = (idx.cpu().sort(-1).values == fx["topk_idx"].sort(-1).values).all(-1)
    assert same.float().mean() >= 0.9
    o, r = out.reshape(T, -1)[same.cuda()].float().cpu(), fx["out"].reshape(T, -1)[same].float()
    eps = torch.finfo(DT).eps
    close = ((o - r).abs() <= 2 * eps * r.abs() + 2 * eps * r.pow(2).mean().sqrt()).all(dim=-1)
    assert close.float().mean() >= 0.9, f"only {close.float().mean():.2f} of the tokens match the literal CPU run"
    assert d.engine.k >= c["k"]


def test_v3_fullsize_fp8_layer(lib_built):
    """One DeepSeek-V3 layer at full size (H=7168, I=2048, E=256, k=8, 8 groups keep 4, scale 2.5, one bf16 shared expert):
    fp8 experts against a bf16 engine holding their dequantised weights.  Same router inputs -> identical routing."""
    from moe_infinity_b200.fp8 import dequantize_block128, quantize_block128
    from test_gpu_fp8_experts import _check_same
    H, I, E, k = 7168, 2048, 256, 8
    a = _v3_engine(E, k, H, 8, 4, True, I=I, num_slots=E, shared_inter=I, gate_dtype=torch.float32, max_tokens=512,
                   expert_dtype=torch.float8_e4m3fn)
    b = _v3_engine(E, k, H, 8, 4, True, I=I, num_slots=E, shared_inter=I, gate_dtype=torch.float32, max_tokens=512,
                   pack_weights=False)
    gen = torch.Generator(device="cuda").manual_seed(3)
    for e in range(E):
        ws = [torch.randn(shp, device="cuda", generator=gen).mul_(0.02).to(DT) for shp in ((I, H), (I, H), (H, I))]
        qs, ss = zip(*[quantize_block128(w) for w in ws])
        a.load_expert(0, e, qs, scales=ss)
        b.load_expert(0, e, [dequantize_block128(q, s) for q, s in zip(qs, ss)])
    shared = [torch.randn(shp, device="cuda", generator=gen).mul_(0.02).to(DT).cpu() for shp in ((I, H), (I, H), (H, I))]
    gate = torch.randn(E, H, device="cuda", generator=gen) * (1.0 / H ** 0.5)
    bias = torch.randn(E, device="cuda", generator=gen) * 0.1
    for eng in (a, b):
        eng.register_shared(0, shared)
        eng.set_gate(0, gate)
        eng.set_gate_bias(0, bias)
    for T in (1, 8, 64, 512):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        _check_same(a, b, x, f"T={T}")
        a.route(0, x); torch.cuda.synchronize()
        ia, wa = a.ws("topk_idx", T).clone(), a.ws("topk_w", T).clone()
        b.route(0, x); torch.cuda.synchronize()
        assert torch.equal(ia, b.ws("topk_idx", T)) and torch.equal(wa, b.ws("topk_w", T)), f"T={T}: routing differs"
        assert (ia >= 0).all() and (ia < E).all()
    a.close(); b.close()


def test_v3_graph_capture_replays_eager(lib_built):
    from moe_infinity_b200 import DecodeSession
    L_, E, k, H, I, T = 3, 64, 8, 256, 256, 8
    eng = _v3_engine(E, k, H, 8, 4, True, I=I, L_=L_, num_slots=L_ * E, shared_inter=I, max_tokens=16)
    torch.manual_seed(0)
    for l in range(L_):
        for e in range(E):
            eng.load_expert(l, e).normal_(0, 0.05)
        eng.register_shared(l, [torch.randn(I, H) * 0.05, torch.randn(I, H) * 0.05, torch.randn(H, I) * 0.05])
        eng.set_gate(l, torch.randn(E, H) * 0.1)
        eng.set_gate_bias(l, torch.randn(E) * 0.1 - 0.2 * l)
    sess = DecodeSession(eng, T).capture()
    for it in range(3):
        sess.x_host.copy_(torch.randn(L_, T, H).to(DT))
        out = sess.step().clone()
        for l in range(L_):
            want = eng.forward(l, sess.x_host[l].cuda())
            torch.cuda.synchronize()
            assert torch.equal(out[l].cuda(), want), (it, l)
    assert eng.stats()["host_syncs"] == 0
    eng.close()


def test_v3_lookahead_uses_next_layers_bias(lib_built):
    """Offload context with lookahead_prefetch=2: the prediction made during layer l is the V3 routing of layer l+1's gate
    and bias applied to layer l's input.  Inputs and gate rows are small integers, so the fp32 logits are exact on both
    sides; the biases are large enough to change the choice against plain top-k of the logits."""
    from moe_infinity_b200 import _lib as L
    Ln, E, k, H, I, T = 3, 16, 4, 128, 128, 6
    eng = _v3_engine(E, k, H, 4, 2, True, I=I, L_=Ln, num_slots=20, lookahead_prefetch=True, gate_dtype=torch.float32,
                     max_tokens=16)
    g = torch.Generator().manual_seed(11)
    for l in range(Ln):
        for e in range(E):
            eng.register_expert(l, e, [torch.randn(I, H, generator=g) * 0.05, torch.randn(I, H, generator=g) * 0.05,
                                       torch.randn(H, I, generator=g) * 0.05])
    gates = [torch.randint(-2, 3, (E, H), generator=g).float() * 0.25 for _ in range(Ln)]
    biases = [torch.randn(E, generator=g) * 0.3 for _ in range(Ln)]
    for l in range(Ln):
        eng.set_gate(l, gates[l])
        eng.set_gate_bias(l, biases[l])
    assert eng.router == L.ROUTER_DEEPSEEK_V3
    differs = 0
    for l in range(Ln - 1):
        x = torch.randint(-2, 3, (T, H), generator=g).to(DT) * 0.5
        eng.forward(l, x.cuda())
        torch.cuda.synchronize()
        look = eng.last_lookahead()
        logits = x.float() @ gates[l + 1].t()
        r = V3.deepseek_v3_route(logits, biases[l + 1], k, 4, 2, True, 2.5)
        want = torch.bincount(r.topk_idx.flatten(), minlength=E).tolist()
        assert look == want, (l, look, want)
        plain = torch.bincount(logits.topk(k, dim=-1).indices.flatten(), minlength=E).tolist()
        differs += plain != want
    assert differs > 0, "the biases never changed the prediction: the test would not notice a bias-free predictor"
    eng.close()


def _tiny_v3():
    from transformers import DeepseekV3Config, DeepseekV3ForCausalLM
    cfg = DeepseekV3Config(vocab_size=512, hidden_size=256, intermediate_size=512, moe_intermediate_size=128,
                           num_hidden_layers=2, first_k_dense_replace=1, num_attention_heads=4, num_key_value_heads=4,
                           n_routed_experts=16, num_experts_per_tok=4, n_group=4, topk_group=2, n_shared_experts=1,
                           routed_scaling_factor=2.5, norm_topk_prob=True, q_lora_rank=64, kv_lora_rank=32,
                           qk_rope_head_dim=16, qk_nope_head_dim=32, v_head_dim=32, max_position_embeddings=128)
    torch.manual_seed(0)
    model = DeepseekV3ForCausalLM(cfg).to(DT).cuda().eval()
    with torch.no_grad():      # tiny init gives near-uniform routing: spread the router, and give it a non-zero bias
        for layer in model.model.layers[1:]:
            layer.mlp.gate.weight.mul_(20.0)
            layer.mlp.gate.e_score_correction_bias.copy_(torch.randn(16) * 0.1)
    return model


def test_patched_deepseek_v3_matches_hf(lib_built):
    from moe_infinity_b200.hf import patch_deepseek_v3
    ref = _tiny_v3()
    ours = copy.deepcopy(ref)
    eng = patch_deepseek_v3(ours, max_tokens=256)
    assert type(ours.model.layers[0].mlp).__name__ == "DeepseekV3MLP"          # the dense layer stays
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


def test_patch_deepseek_v3_refuses_single_normalised_expert(lib_built):
    from transformers import DeepseekV3Config, DeepseekV3ForCausalLM
    from moe_infinity_b200.hf import patch_deepseek_v3
    cfg = DeepseekV3Config(vocab_size=64, hidden_size=64, intermediate_size=128, moe_intermediate_size=64,
                           num_hidden_layers=2, first_k_dense_replace=1, num_attention_heads=2, num_key_value_heads=2,
                           n_routed_experts=8, num_experts_per_tok=1, n_group=1, topk_group=1, norm_topk_prob=True,
                           q_lora_rank=32, kv_lora_rank=16, qk_rope_head_dim=8, qk_nope_head_dim=16, v_head_dim=16)
    with pytest.raises(ValueError, match="num_experts_per_tok == 1"):
        patch_deepseek_v3(DeepseekV3ForCausalLM(cfg))
