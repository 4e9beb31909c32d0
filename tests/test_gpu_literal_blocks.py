"""GPU: the reference's OWN, unmodified MoE blocks (moe_infinity/models/{mixtral,deepseek,switch_transformers,nllb_moe}.py, loaded
through tests/shims/ref_loader.py from a reference checkout or its byte-compiled staging oracle/_ref/pyref; skipped where neither exists) running on the GPU on
top of this repository's plugin objects, constructed exactly the way moe_infinity/runtime/model_offload.py constructs the
reference's (`prefetch_handle(prefix, ratio)`, `expert_dispatcher(E, L, dtype, expert_type, num_threads)` -- five positional
arguments, :143-145, :471-477 -- then `offload` / `register_expert` / `set_expert_dispatcher`).  The block's Python (router
math, mask build, combine loop) is the reference's; everything behind `expert_executor.dispatch_local` is libb2m.so.
Results are held to the golden vectors the same literal blocks produced on CPU (tests/golden/*.pt)."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

import ref_loader  # noqa: E402
from test_gpu_parity import hidden_close, load_case  # noqa: E402

needs_reference = pytest.mark.skipif(not ref_loader.available(), reason="neither /root/reference nor oracle/_ref/pyref present")


def _plugin(c, expert_type, dtype_int, layers=1):
    """The three objects OffloadEngine builds (model_offload.py:143-160, 471-477), reference signatures only."""
    from moe_infinity_b200.compat import DistributedExpertExecutor, expert_dispatcher, prefetch_handle
    h = prefetch_handle("/tmp/b2m_literal_unused", 0.9)
    d = expert_dispatcher(c["E"], layers, dtype_int, expert_type, 8)
    assert d.handle is h
    tid = 0
    for e in range(c["E"]):
        ids = []
        for w in c["experts"][e]:                      # named_parameters order
            h.offload(w, tid)
            ids.append(tid)
            tid += 1
        d.register_expert(0, e, ids)                   # model_offload.py:851-853
    ex = DistributedExpertExecutor()
    ex.set_expert_dispatcher(d)
    return h, d, ex


@needs_reference
@pytest.mark.parametrize("name", ["mixtral_mini_bf16", "mixtral_ragged_bf16", "mixtral_mini_f16", "mixtral_onetoken_bf16"])
def test_literal_mixtral_block_on_gpu(lib_built, name):
    from moe_infinity_b200 import _lib as L
    ns = ref_loader.load()
    c, fx = load_case(name)
    dt = c["dtype"]
    cfg = types.SimpleNamespace(hidden_size=c["H"], intermediate_size=c["I"], num_local_experts=c["E"],
                                num_experts_per_tok=c["k"], hidden_act="silu")
    blk = ns.mixtral.SyncMixtralSparseMoeBlock(cfg).to(dt)
    with torch.no_grad():
        blk.gate.weight.copy_(c["gate"])
    blk.gate.cuda()                                     # dense parameters live on the device; experts stay with the engine
    _, d, ex = _plugin(c, L.EXPERT_MIXTRAL, L.DTYPE_BF16 if dt == torch.bfloat16 else L.DTYPE_F16)
    blk.expert_executor, blk.layer_id = ex, 0
    with torch.no_grad():
        out, logits = blk(c["hidden"].cuda())
    torch.cuda.synchronize()
    assert out.shape == c["hidden"].shape and out.dtype == dt and out.is_cuda
    T = c["B"] * c["S"]
    same = (logits.cpu() == fx["router_logits"]).all(dim=-1) & ~fx["tied"]    # GPU vs CPU gate GEMM may round differently
    assert same.float().mean() > 0.9 or T == 1
    if bool(same.any()):
        hidden_close(out.reshape(T, -1)[same.cuda()], fx["out"].reshape(T, -1)[same], None, dt, "literal mixtral block")
    assert d.engine.k == c["k"]                         # top_k learnt from the masks


@needs_reference
@pytest.mark.parametrize("name", ["deepseek_mini_bf16", "deepseek_group_bf16"])
def test_literal_deepseek_block_on_gpu(lib_built, name):
    """deepseek.py:8-137 with the literal MoEGate: top-k 4 masks reach a dispatcher that was built without a top_k."""
    from moe_infinity_b200 import _lib as L
    ns = ref_loader.load()
    c, fx = load_case(name)
    dt = c["dtype"]
    cf = fx["cfg"]
    cfg = types.SimpleNamespace(model_type="deepseek_v2", hidden_size=c["H"], intermediate_size=c["I"] * 4,
                                moe_intermediate_size=c["I"], n_routed_experts=c["E"], num_experts_per_tok=c["k"],
                                n_shared_experts=cf["n_shared"], routed_scaling_factor=cf["routed_scaling_factor"],
                                scoring_func="softmax", aux_loss_alpha=0.0, seq_aux=False, topk_method=cf["topk_method"],
                                n_group=cf["n_group"], topk_group=cf["topk_group"], norm_topk_prob=cf["norm_topk_prob"],
                                hidden_act="silu", pretraining_tp=1)
    blk = ns.deepseek.DeepseekMoEBlock(cfg).to(dt)
    blk.eval()
    with torch.no_grad():
        blk.gate.weight.copy_(c["gate"])
        if cf["n_shared"] is not None:
            blk.shared_experts.gate_proj.weight.copy_(c["shared"][0])
            blk.shared_experts.up_proj.weight.copy_(c["shared"][1])
            blk.shared_experts.down_proj.weight.copy_(c["shared"][2])
    blk.gate.cuda()
    if cf["n_shared"] is not None:
        blk.shared_experts.cuda()                        # plain nn.Module in the reference too (deepseek.py:133-136)
    _, d, ex = _plugin(c, L.EXPERT_DEEPSEEK, L.DTYPE_BF16)
    blk.expert_executor, blk.layer_id = ex, 0
    with torch.no_grad():
        out = blk(c["hidden"].cuda())
    torch.cuda.synchronize()
    T = c["B"] * c["S"]
    ok = ~fx["tied"]
    o, r = out.reshape(T, -1)[ok.cuda()].float().cpu(), fx["out"].reshape(T, -1)[ok].float()
    eps = torch.finfo(dt).eps
    # the literal gate runs as a GPU fp32 GEMM here (CPU in the fixture): scores differ in the last fp32 bits, which can
    # flip a near-tied expert choice -> compare the tokens whose output agrees to the rounding bound and demand most do
    close = ((o - r).abs() <= 2 * eps * r.abs() + 2 * eps * r.pow(2).mean().sqrt()).all(dim=-1)
    assert close.float().mean() >= 0.9, f"only {close.float().mean():.2f} of the untied tokens match the literal CPU run"
    assert d.engine.k >= c["k"]


@needs_reference
@pytest.mark.parametrize("name", ["switch_mini_bf16"])
def test_literal_switch_block_on_gpu(lib_built, name):
    """switch_transformers.py:41-113 on the 4.x-order router shim; capacity-dropped tokens pass through unchanged."""
    from transformers import SwitchTransformersConfig
    from moe_infinity_b200 import _lib as L
    ns = ref_loader.load()
    c, fx = load_case(name)
    dt = c["dtype"]
    cfg = SwitchTransformersConfig(d_model=c["H"], d_ff=c["I"], num_experts=c["E"], expert_capacity=c["capacity"],
                                   router_bias=False, router_jitter_noise=0.0, router_dtype="float32", dropout_rate=0.0,
                                   dense_act_fn="relu", num_layers=1, num_sparse_encoder_layers=1)
    blk = ns.switch.SyncSwitchTransformersSparseMLP(cfg).to(dt)
    blk.eval()
    with torch.no_grad():
        blk.router.classifier.weight.copy_(c["gate"])
    blk.router.cuda()
    _, d, ex = _plugin(c, L.EXPERT_SWITCH, L.DTYPE_BF16)
    blk.expert_executor, blk.layer_id = ex, 0
    with torch.no_grad():
        out, (logits, expert_index) = blk(c["hidden"].cuda())
    torch.cuda.synchronize()
    assert out.shape == c["hidden"].shape
    stable = (logits.float().cpu().reshape(-1, c["E"]) - fx["router_logits"].float().reshape(-1, c["E"])).abs().max(-1).values < 1e-4
    assert stable.float().mean() > 0.9
    assert torch.equal(expert_index.cpu().flatten()[stable], fx["expert_index"].flatten()[stable])
    hidden_close(out, fx["out"], None, dt, "literal switch block")


@needs_reference
@pytest.mark.parametrize("name", ["nllb_mini_bf16", "nllb_capacity_f16"])
def test_literal_nllb_block_on_gpu(lib_built, name):
    """nllb_moe.py:20-115 (HF top-2 router on its 4.x contract, 3-D hidden states and masks handed to dispatch_local, bias
    experts fc1|fc1_bias|fc2|fc2_bias, tokens dropped by the router's capacity pass through) on top of the plugin objects."""
    import make_golden as G
    from moe_infinity_b200 import _lib as L
    ns = ref_loader.load()
    if not hasattr(ns, "nllb"):
        pytest.skip("the NLLB block could not be imported")
    fx = torch.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", name + ".pt"), weights_only=False)
    c = G.build_nllb(name)
    assert torch.equal(c["hidden"], fx["hidden"])
    dt = c["dtype"]
    blk = ns.nllb.SyncNllbMoeSparseMLP(G.nllb_config(c["H"], c["I"], c["E"], c["capacity"]), c["I"]).to(dt)
    blk.eval()
    with torch.no_grad():
        blk.router.classifier.weight.copy_(c["gate"])
    blk.router.cuda()
    _, d, ex = _plugin(c, L.EXPERT_NLLB, L.DTYPE_BF16 if dt == torch.bfloat16 else L.DTYPE_F16)
    blk.expert_executor, blk.layer_id = ex, 0
    with torch.no_grad():
        out, (probs, top1) = blk(c["hidden"].cuda())
    torch.cuda.synchronize()
    assert out.shape == c["hidden"].shape and out.dtype == dt and out.is_cuda
    T = c["B"] * c["S"]
    # the router runs in fp32 on the GPU vs on the CPU for the fixture: keep the tokens whose combining weights agree exactly
    same = (probs.cpu().reshape(T, -1) == fx["router_probs"].reshape(T, -1)).all(dim=-1)
    assert same.float().mean() > 0.7
    hidden_close(out.reshape(T, -1)[same.cuda()], fx["out"].reshape(T, -1)[same], None, dt, "literal nllb block")
    assert torch.equal(top1.cpu()[same], fx["top1"][same])
