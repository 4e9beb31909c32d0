"""HuggingFace plug-in helpers: run a `transformers` Mixtral, DeepSeek-V3, Qwen2-MoE, Qwen3-MoE or Llama 4 model with its MoE
blocks executed by the CUDA engine (`patch_mixtral`, `patch_deepseek_v3`, `patch_qwen_moe`, `patch_llama4`), and load the
routed experts of a published AWQ / GPTQ 4-bit checkpoint into an f16 int4 engine (`load_int4_checkpoint`) or of a published
FP8 checkpoint into an fp8 engine (`load_fp8_checkpoint`) as they are stored.

The reference achieves this by monkey-patching HF classes at load time (moe_infinity/runtime/model_offload.py:285-321:
`MixtralSparseMoeBlock -> SyncMixtralSparseMoeBlock`).  The installed transformers (5.x) stores the experts of a layer as
fused 3-D parameters (`MixtralExperts.gate_up_proj [E, 2I, H]`, `down_proj [E, H, I]`) and its block returns the hidden
states only, so this helper swaps `layer.mlp` for an adapter with that signature; the adapter keeps the router GEMM in
PyTorch (same logits as HF) and hands everything after it to `MoEEngine.forward`.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Optional, Sequence, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import fp8 as F8
from . import int4 as I4
from .engine import MoEEngine


def _load(engine: MoEEngine, layer: int, expert: int, ws, resident: bool):
    """Hand one expert's bf16 matrices to `engine`, quantised first when the engine stores fp8 (`fp8.quantize_block128`, or
    `fp8.quantize_row` for fp8_scales="row") or int4 (`int4.quantize_g128`, with scales of the engine's dtype) experts."""
    kw = {}
    if engine.fp8:
        quantize = F8.quantize_row if engine.fp8_scales == "row" else F8.quantize_block128
        ws, scales = zip(*[quantize(w) for w in ws])
        kw = dict(scales=scales)
    elif engine.int4:
        ws, scales, zeros = zip(*[I4.quantize_g128(w, scale_dtype=engine.dtype) for w in ws])
        kw = dict(scales=scales, zeros=zeros)
    if resident:
        engine.load_expert(layer, expert, ws, **kw)
    else:
        engine.register_expert(layer, expert, ws, **kw)


class B200MixtralMoeAdapter(nn.Module):
    """Drop-in for transformers>=5 `MixtralSparseMoeBlock`: forward(hidden[B,S,H]) -> hidden[B,S,H]."""

    def __init__(self, engine: MoEEngine, layer_id: int, gate_weight: torch.Tensor):
        super().__init__()
        self.engine = engine
        self.layer_id = layer_id
        self.gate_weight = nn.Parameter(gate_weight.detach().clone(), requires_grad=False)

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        shape = hidden_states.shape
        x = hidden_states.reshape(-1, shape[-1])
        router_logits = F.linear(x, self.gate_weight)      # same GEMM HF's MixtralTopKRouter runs
        out = self.engine.forward(self.layer_id, x, router_logits=router_logits)
        return out.reshape(shape)


def patch_mixtral(model, max_tokens: int = 4096, num_slots: int = 0, device_memory_ratio: float = 0.0,
                  resident: bool = True, engine: Optional[MoEEngine] = None) -> MoEEngine:
    """Move every expert of `model` (a transformers MixtralForCausalLM / MixtralModel on a CUDA device) into a
    MoEEngine and replace the MoE blocks.  `resident=False` registers experts as pinned host blobs (offload mode,
    budget from num_slots / device_memory_ratio) instead of loading all of them into HBM.  `engine` may be given (built with
    the model's shapes), e.g. one with expert_dtype=torch.uint4: the experts are then quantised with `int4.quantize_g128`."""
    cfg = model.config
    layers = model.model.layers if hasattr(model, "model") else model.layers
    dev = next(model.parameters()).device
    dtype = next(model.parameters()).dtype
    L, E, H, I, k = len(layers), cfg.num_local_experts, cfg.hidden_size, cfg.intermediate_size, cfg.num_experts_per_tok
    if engine is None:
        engine = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, max_tokens=max_tokens,
                           num_slots=(L * E if resident and not num_slots else num_slots),
                           device_memory_ratio=device_memory_ratio, device=dev.index or 0)
    for l, layer in enumerate(layers):
        moe = layer.mlp
        gu, dn = moe.experts.gate_up_proj.data, moe.experts.down_proj.data     # [E,2I,H], [E,H,I]
        for e in range(E):
            w1, w3, w2 = gu[e, :I], gu[e, I:], dn[e]                            # reference order: w1 | w2 | w3
            _load(engine, l, e, [w1, w2, w3], resident)
        layer.mlp = B200MixtralMoeAdapter(engine, l, moe.gate.weight.data)
    return engine


class B200DeepseekV3MoeAdapter(nn.Module):
    """Drop-in for transformers>=5 `DeepseekV3MoE`: forward(hidden[B,S,H]) -> hidden[B,S,H].  The router (fp32 gate GEMM,
    sigmoid, correction bias, group selection, weights), the routed experts, the shared expert and the combine all run in
    the engine (fused gate, router_in_kind 0)."""

    def __init__(self, engine: MoEEngine, layer_id: int):
        super().__init__()
        self.engine = engine
        self.layer_id = layer_id

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        shape = hidden_states.shape
        out = self.engine.forward(self.layer_id, hidden_states.reshape(-1, shape[-1]))
        return out.reshape(shape)


def patch_deepseek_v3(model, max_tokens: int = 4096, num_slots: int = 0, device_memory_ratio: float = 0.0,
                      resident: bool = True, engine: Optional[MoEEngine] = None) -> MoEEngine:
    """Move the routed experts, shared experts, router weights and correction biases of `model` (a transformers
    DeepseekV3ForCausalLM / DeepseekV3Model on a CUDA device) into a MoEEngine (ROUTER_DEEPSEEK_V3) and replace its MoE
    blocks (layers >= config.first_k_dense_replace; the dense layers before them stay as they are).  `engine` may be
    given (built with router=ROUTER_DEEPSEEK_V3 and the model's shapes), e.g. one with expert_dtype=torch.float8_e4m3fn or
    torch.uint4: the experts are then quantised with `fp8.quantize_block128` or `int4.quantize_g128`.  `resident=False` registers experts as pinned host
    blobs (offload mode, budget from num_slots / device_memory_ratio)."""
    cfg = model.config
    if cfg.num_experts_per_tok == 1 and cfg.norm_topk_prob:
        # transformers normalises a single weight to 1 here; the reference gate (and this engine) only normalise for k > 1
        raise ValueError("num_experts_per_tok == 1 with norm_topk_prob: transformers and the reference gate disagree")
    layers = model.model.layers if hasattr(model, "model") else model.layers
    dev = next(model.parameters()).device
    dtype = next(model.parameters()).dtype
    L_, E, H, I, k = len(layers), cfg.n_routed_experts, cfg.hidden_size, cfg.moe_intermediate_size, cfg.num_experts_per_tok
    moe_layers = [l for l in range(L_) if l >= cfg.first_k_dense_replace]
    if engine is None:
        engine = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                           router=L.ROUTER_DEEPSEEK_V3, max_tokens=max_tokens, num_slots=(L_ * E if resident and not num_slots else num_slots),
                           device_memory_ratio=device_memory_ratio, shared_inter=I * cfg.n_shared_experts, n_group=cfg.n_group,
                           topk_group=cfg.topk_group, norm_topk_prob=cfg.norm_topk_prob,
                           routed_scaling_factor=cfg.routed_scaling_factor, gate_dtype=torch.float32, device=dev.index or 0)
    elif engine.router != L.ROUTER_DEEPSEEK_V3:
        raise ValueError("patch_deepseek_v3 needs an engine built with router=ROUTER_DEEPSEEK_V3")
    for l in moe_layers:
        moe = layers[l].mlp
        gu, dn = moe.experts.gate_up_proj.data, moe.experts.down_proj.data     # [E,2I,H], [E,H,I]
        for e in range(E):
            _load(engine, l, e, [gu[e, :I], gu[e, I:], dn[e]], resident)     # DeepSeek order: gate | up | down
        sh = moe.shared_experts
        engine.register_shared(l, [sh.gate_proj.weight.data, sh.up_proj.weight.data, sh.down_proj.weight.data])
        engine.set_gate(l, moe.gate.weight.data)
        engine.set_gate_bias(l, moe.gate.e_score_correction_bias.data)
        layers[l].mlp = B200DeepseekV3MoeAdapter(engine, l)
    return engine


class B200QwenMoeAdapter(nn.Module):
    """Drop-in for transformers>=5 `Qwen2MoeSparseMoeBlock` / `Qwen3MoeSparseMoeBlock`: forward(hidden[B,S,H]) ->
    hidden[B,S,H].  The router GEMM stays in PyTorch (`F.linear` in the model dtype, the logits HF's Qwen2MoeTopKRouter
    computes); the softmax, top-k, weights, routed experts, gated shared expert (Qwen2) and the combine run in the engine."""

    def __init__(self, engine: MoEEngine, layer_id: int, gate_weight: torch.Tensor):
        super().__init__()
        self.engine = engine
        self.layer_id = layer_id
        self.gate_weight = nn.Parameter(gate_weight.detach().clone(), requires_grad=False)

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        shape = hidden_states.shape
        x = hidden_states.reshape(-1, shape[-1])
        router_logits = F.linear(x, self.gate_weight)
        out = self.engine.forward(self.layer_id, x, router_logits=router_logits)
        return out.reshape(shape)


def _is_qwen_sparse_block(mlp) -> bool:
    return hasattr(mlp, "experts") and hasattr(mlp, "gate") and hasattr(mlp.experts, "gate_up_proj")


def patch_qwen_moe(model, max_tokens: int = 4096, num_slots: int = 0, device_memory_ratio: float = 0.0,
                   resident: bool = True, engine: Optional[MoEEngine] = None) -> MoEEngine:
    """Move the routed experts, shared experts and shared-expert gates (Qwen2-MoE) of `model` (a transformers
    Qwen2MoeForCausalLM or Qwen3MoeForCausalLM, or their base models, on a CUDA device) into a MoEEngine
    (ROUTER_QWEN_MOE, gate|up|down experts) and replace its sparse MoE blocks.  Only layers whose `mlp` is the sparse block
    are replaced, so `mlp_only_layers` and `decoder_sparse_step` keep their dense MLPs.  `engine` may be given (built with
    router=ROUTER_QWEN_MOE and the model's shapes), e.g. one with expert_dtype=torch.float8_e4m3fn or torch.uint4: the
    routed experts are then quantised with `fp8.quantize_block128` or `int4.quantize_g128`; shared experts stay in the
    model dtype.  `resident=False` registers the routed experts as pinned host blobs (offload mode, budget from num_slots /
    device_memory_ratio)."""
    cfg = model.config
    layers = model.model.layers if hasattr(model, "model") else model.layers
    dev = next(model.parameters()).device
    dtype = next(model.parameters()).dtype
    L_, E, H, I, k = len(layers), cfg.num_experts, cfg.hidden_size, cfg.moe_intermediate_size, cfg.num_experts_per_tok
    moe_layers = [l for l in range(L_) if _is_qwen_sparse_block(layers[l].mlp)]
    shared = bool(moe_layers) and hasattr(layers[moe_layers[0]].mlp, "shared_expert")
    shared_inter = cfg.shared_expert_intermediate_size if shared else 0
    if engine is None:
        engine = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                           router=L.ROUTER_QWEN_MOE, max_tokens=max_tokens,
                           num_slots=(L_ * E if resident and not num_slots else num_slots),
                           device_memory_ratio=device_memory_ratio, shared_inter=shared_inter,
                           norm_topk_prob=bool(cfg.norm_topk_prob), device=dev.index or 0)
    elif engine.router != L.ROUTER_QWEN_MOE or engine.expert_type != L.EXPERT_DEEPSEEK:
        raise ValueError("patch_qwen_moe needs an engine built with router=ROUTER_QWEN_MOE and expert_type=EXPERT_DEEPSEEK")
    elif engine.shared_inter != shared_inter:
        raise ValueError(f"the engine's shared_inter {engine.shared_inter} does not match the model's {shared_inter}")
    for l in moe_layers:
        moe = layers[l].mlp
        gu, dn = moe.experts.gate_up_proj.data, moe.experts.down_proj.data     # [E,2I,H], [E,H,I]
        for e in range(E):
            _load(engine, l, e, [gu[e, :I], gu[e, I:], dn[e]], resident)     # HF order: gate | up | down
        if shared:
            sh = moe.shared_expert
            engine.register_shared(l, [sh.gate_proj.weight.data, sh.up_proj.weight.data, sh.down_proj.weight.data])
            engine.set_shared_gate(l, moe.shared_expert_gate.weight.data)
        layers[l].mlp = B200QwenMoeAdapter(engine, l, moe.gate.weight.data)
    return engine


class B200Llama4MoeAdapter(nn.Module):
    """Drop-in for transformers>=5 `Llama4TextMoe`: forward(hidden[..., H]) -> (out [T, H], router_logits [T, E]), the
    tuple the Llama 4 decoder layer unpacks.  The router GEMM stays in PyTorch (`F.linear` in the model dtype, the logits
    HF's Llama4Router computes and returns); the top-k, the sigmoid weights, the scaling of the expert inputs, the routed
    experts, the shared expert and the combine run in the engine."""

    def __init__(self, engine: MoEEngine, layer_id: int, gate_weight: torch.Tensor):
        super().__init__()
        self.engine = engine
        self.layer_id = layer_id
        self.gate_weight = nn.Parameter(gate_weight.detach().clone(), requires_grad=False)

    def forward(self, hidden_states: torch.Tensor):
        x = hidden_states.reshape(-1, hidden_states.shape[-1])
        router_logits = F.linear(x, self.gate_weight)
        return self.engine.forward(self.layer_id, x, router_logits=router_logits), router_logits


def _is_llama4_moe(ff) -> bool:
    try:
        from transformers.models.llama4.modeling_llama4 import Llama4TextMoe
    except ImportError:
        return False
    return isinstance(ff, Llama4TextMoe)


def patch_llama4(model, max_tokens: int = 4096, num_slots: int = 0, device_memory_ratio: float = 0.0,
                 resident: bool = True, engine: Optional[MoEEngine] = None) -> MoEEngine:
    """Move the routed and shared experts of `model` (a transformers>=5 Llama4ForCausalLM, or the text model of a
    Llama4ForConditionalGeneration, on a CUDA device) into a MoEEngine (ROUTER_LLAMA4, gate|up|down experts) and replace
    its `Llama4TextMoe` blocks.  Only layers whose `feed_forward` is that block are replaced, so the dense layers Maverick
    interleaves (`interleave_moe_layer_step`) stay.  Llama4TextExperts stores an expert's weights fused and transposed:
    gate = gate_up_proj[e][:, :I].T, up = gate_up_proj[e][:, I:].T, down = down_proj[e].T.  `engine` may be given (built
    with router=ROUTER_LLAMA4 and the model's shapes), e.g. one with expert_dtype=torch.float8_e4m3fn or torch.uint4: the
    routed experts are then quantised with `fp8.quantize_block128` or `int4.quantize_g128`; the shared experts stay in the
    model dtype.  `resident=False` registers the routed experts as pinned host blobs (offload mode, budget from num_slots
    / device_memory_ratio)."""
    cfg = model.config
    cfg = getattr(cfg, "text_config", cfg)
    layers = model.model.layers if hasattr(model, "model") else model.layers
    dev = next(model.parameters()).device
    dtype = next(model.parameters()).dtype
    L_, E, H, I, k = len(layers), cfg.num_local_experts, cfg.hidden_size, cfg.intermediate_size, cfg.num_experts_per_tok
    moe_layers = [l for l in range(L_) if _is_llama4_moe(layers[l].feed_forward)]
    if engine is None:
        engine = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                           router=L.ROUTER_LLAMA4, max_tokens=max_tokens,
                           num_slots=(L_ * E if resident and not num_slots else num_slots),
                           device_memory_ratio=device_memory_ratio, shared_inter=I, device=dev.index or 0)
    elif engine.router != L.ROUTER_LLAMA4 or engine.expert_type != L.EXPERT_DEEPSEEK:
        raise ValueError("patch_llama4 needs an engine built with router=ROUTER_LLAMA4 and expert_type=EXPERT_DEEPSEEK")
    elif engine.shared_inter != I:
        raise ValueError(f"the engine's shared_inter {engine.shared_inter} does not match the model's shared expert ({I})")
    for l in moe_layers:
        moe = layers[l].feed_forward
        gu, dn = moe.experts.gate_up_proj.data, moe.experts.down_proj.data     # [E,H,2I], [E,I,H]
        for e in range(E):
            _load(engine, l, e, [gu[e, :, :I].t().contiguous(), gu[e, :, I:].t().contiguous(), dn[e].t().contiguous()],
                  resident)
        sh = moe.shared_expert
        engine.register_shared(l, [sh.gate_proj.weight.data, sh.up_proj.weight.data, sh.down_proj.weight.data])
        layers[l].feed_forward = B200Llama4MoeAdapter(engine, l, moe.router.weight.data)
    return engine


# ---------------------------------------------------------------- published AWQ / GPTQ checkpoints
def _int4_method(qc: dict) -> str:
    """Validate a checkpoint's `quantization_config` and return "awq", "gptq" or "gptq_v2"."""
    method = str(qc.get("quant_method", "")).lower()
    bits = qc.get("bits", qc.get("w_bit"))
    group = qc.get("group_size", qc.get("q_group_size"))
    if method not in ("awq", "gptq"):
        raise ValueError(f"quant_method {method!r}: only 'awq' and 'gptq' 4-bit checkpoints are supported")
    if bits != 4:
        raise ValueError(f"{method} checkpoint with bits={bits}: only 4-bit weights are supported")
    if group != I4.GROUP:
        raise ValueError(f"{method} checkpoint with group_size={group}: only group size {I4.GROUP} is supported")
    if method == "awq":
        if not qc.get("zero_point", True):
            raise ValueError("AWQ checkpoint with zero_point=false: only asymmetric (zero-point) AWQ is supported")
        version = str(qc.get("version", "gemm")).lower()
        if version != "gemm":
            raise ValueError(f"AWQ checkpoint version {version!r}: only the 'gemm' packing is supported")
        return "awq"
    fmt = str(qc.get("checkpoint_format", "gptq")).lower()
    if fmt not in ("gptq", "gptq_v2"):
        raise ValueError(f"GPTQ checkpoint_format {fmt!r}: only 'gptq' and 'gptq_v2' are supported")
    return fmt


def load_int4_checkpoint(engine: MoEEngine, shards: Union[str, Sequence[str]], quantization_config: dict, model_type: str,
                         resident: bool = True, act_order: bool = False) -> List[int]:
    """Load the routed experts and router weights of a published AWQ or GPTQ 4-bit checkpoint (its safetensors `shards`,
    its config's `quantization_config`, `model_type` "mixtral", "deepseek_v2" / "deepseek_v3" or "qwen2_moe" / "qwen3_moe")
    into `engine`, an int4
    engine with float16 activations (`MoEEngine(dtype=torch.float16, expert_dtype=torch.uint4)`), without changing a
    weight (`int4.from_awq` / `int4.from_gptq`).  Tensors are read one at a time with `safetensors.safe_open`.

    Mixtral: model.layers.{l}.block_sparse_moe.experts.{e}.w{1,2,3}.* and ...block_sparse_moe.gate.weight.  DeepSeek:
    model.layers.{l}.mlp.experts.{e}.{gate,up,down}_proj.*, mlp.gate.weight (and mlp.gate.e_score_correction_bias for a V3
    router) and mlp.shared_experts.*, whose dequantised weights are registered as the f16 shared expert; layers without
    experts (no mlp.gate.weight) are skipped.  Qwen2-MoE / Qwen3-MoE (an engine with router=ROUTER_QWEN_MOE): the same
    routed-expert and router names, mlp.shared_expert.{gate,up,down}_proj.* for the shared expert (dequantised to f16) and
    the plain mlp.shared_expert_gate.weight for its gate (a checkpoint holding only a quantised form of that gate is
    refused).  `resident=False` registers the experts as pinned host blobs (offload).
    act_order=True loads act-order GPTQ (desc_act, a g_idx other than c // 128) as well, without changing a weight: per
    expert, P = the gate/up order and P2 = the down projection's (`int4.from_gptq_act_order`); the engine stores
    gate/up as W[P2][:, P] and down as W[:, P2] (so the gate/up GEMM writes h[P2], which the down projection consumes),
    and each layer with a non-identity P gets one [E, H] gather table (`MoEEngine.set_input_perm`).  The gate and up
    projections of an expert must share their g_idx (GPTQ derives both from the same input Hessian); a checkpoint where
    they differ is refused, naming the layer and expert.
    Refused with a message: bits other than 4, group sizes other than 128, AWQ without zero points or in a packing other
    than "gemm", act-order GPTQ without act_order=True, and a missing tensor.  Returns the layers it loaded."""
    from safetensors import safe_open

    if not engine.int4 or engine.dtype != torch.float16:
        raise ValueError("load_int4_checkpoint needs an int4 engine with float16 activations "
                         "(MoEEngine(dtype=torch.float16, expert_dtype=torch.uint4))")
    method = _int4_method(quantization_config)
    mixtral = model_type == "mixtral"
    qwen = model_type in ("qwen2_moe", "qwen3_moe")
    if not mixtral and not qwen and not model_type.startswith("deepseek"):
        raise ValueError(f"model_type {model_type!r}: Mixtral, DeepSeek and Qwen-MoE checkpoints are supported")
    if mixtral != (engine.expert_type == L.EXPERT_MIXTRAL):
        raise ValueError(f"model_type {model_type!r} does not match the engine's expert_type {engine.expert_type}")
    if qwen != (engine.router == L.ROUTER_QWEN_MOE):
        raise ValueError(f"model_type {model_type!r} does not match the engine's router {engine.router}")
    shared_name = "shared_expert" if qwen else "shared_experts"
    if isinstance(shards, str):
        shards = [shards]
    parts = ("qweight", "qzeros", "scales")
    with contextlib.ExitStack() as stack:
        files = [stack.enter_context(safe_open(path, framework="pt", device="cpu")) for path in shards]
        where: Dict[str, object] = {k: f for f in files for k in f.keys()}

        def linear(prefix: str):
            """(q, s, z, perm) of one linear layer: (q, s, z) hold W[:, perm]; perm is None for natural column order."""
            t = [where[f"{prefix}.{p}"].get_tensor(f"{prefix}.{p}") for p in parts]
            if method == "awq":
                return (*I4.from_awq(*t), None)
            gi = f"{prefix}.g_idx"
            g_idx = where[gi].get_tensor(gi) if gi in where else None
            if act_order and g_idx is not None:
                q, s_, z, perm = I4.from_gptq_act_order(*t, g_idx, checkpoint_format=method)
                return q, s_, z, (None if torch.equal(perm, torch.arange(perm.numel())) else perm)
            if g_idx is not None and not torch.equal(g_idx.to(torch.int64), torch.arange(g_idx.numel()) // I4.GROUP):
                raise ValueError(f"{prefix}: GPTQ g_idx is not c // 128, an act-order (desc_act) checkpoint: "
                                 "load it with act_order=True")
            return (*I4.from_gptq(*t, g_idx=g_idx, checkpoint_format=method), None)

        def shared(prefix: str) -> torch.Tensor:
            """A shared expert's linear layer dequantised to f16 in its natural column order."""
            q, s_, z, perm = linear(prefix)
            w = I4.dequantize_g128(q, s_, z, torch.float16)
            return w if perm is None else w[:, perm.argsort()]

        def rows(qsz, perm):
            """(q, s, z) with their rows permuted (each row keeps its own scale and zero words)."""
            return tuple(t[perm].contiguous() for t in qsz) if perm is not None else qsz

        if mixtral:
            layers = list(range(engine.L))
            moe = "block_sparse_moe"
            names = ("w1", "w2", "w3")                                 # reference order: w1 | w2 | w3
        else:
            layers = [l for l in range(engine.L) if f"model.layers.{l}.mlp.gate.weight" in where]
            moe = "mlp"
            names = ("gate_proj", "up_proj", "down_proj")              # DeepSeek order: gate | up | down
        need = []
        for l in layers:
            base = f"model.layers.{l}.{moe}"
            need.append(f"{base}.gate.weight")
            need += [f"{base}.experts.{e}.{n}.{p}" for e in range(engine.E) for n in names for p in parts]
            if not mixtral and engine.shared_inter > 0:
                need += [f"{base}.{shared_name}.{n}.{p}" for n in names for p in parts]
            if qwen and engine.shared_inter > 0:
                key = f"{base}.shared_expert_gate"
                if f"{key}.weight" not in where and f"{key}.qweight" in where:
                    raise ValueError(f"the checkpoint stores {key} quantised ({key}.qweight); its plain {key}.weight "
                                     "is needed (the shared-expert gate runs in the model dtype)")
                need.append(f"{key}.weight")
            if not mixtral and engine.router == L.ROUTER_DEEPSEEK_V3:
                need.append(f"{base}.gate.e_score_correction_bias")
        missing = [k for k in need if k not in where]
        if missing:
            raise ValueError(f"the checkpoint has no tensor {missing[0]} ({len(missing)} missing)")
        (g_, u_), d_ = ((0, 2), 1) if mixtral else ((0, 1), 2)   # positions of gate, up and down in `names`
        for l in layers:
            base = f"model.layers.{l}.{moe}"
            table = torch.arange(engine.H).repeat(engine.E, 1)
            for e in range(engine.E):
                mats = [linear(f"{base}.experts.{e}.{n}") for n in names]
                pg, pu, p2 = mats[g_][3], mats[u_][3], mats[d_][3]
                if not (pg is None and pu is None) and (pg is None or pu is None or not torch.equal(pg, pu)):
                    raise ValueError(f"layer {l} expert {e}: {names[g_]} and {names[u_]} have different g_idx; act-order "
                                     "experts must share one input order for both (one permutation of the routed rows)")
                if pg is not None:
                    table[e] = pg
                qsz = [m[:3] for m in mats]
                for i in (g_, u_):
                    qsz[i] = rows(qsz[i], p2)            # gate/up rows in the down projection's input order
                qs, ss, zs = zip(*qsz)
                if resident:
                    engine.load_expert(l, e, qs, scales=ss, zeros=zs)
                else:
                    engine.register_expert(l, e, qs, scales=ss, zeros=zs)
            if act_order and not torch.equal(table, torch.arange(engine.H).expand(engine.E, engine.H)):
                engine.set_input_perm(l, table)
            if not mixtral and engine.shared_inter > 0:
                engine.register_shared(l, [shared(f"{base}.{shared_name}.{n}") for n in names])
            if qwen and engine.shared_inter > 0:
                key = f"{base}.shared_expert_gate.weight"
                engine.set_shared_gate(l, where[key].get_tensor(key).to(engine.dtype))
            key = f"{base}.gate.weight"
            engine.set_gate(l, where[key].get_tensor(key))
            if not mixtral and engine.router == L.ROUTER_DEEPSEEK_V3:
                key = f"{base}.gate.e_score_correction_bias"
                engine.set_gate_bias(l, where[key].get_tensor(key).float())
    return layers


# ---------------------------------------------------------------- published FP8 checkpoints
def _fp8_layout(qc: dict):
    """Validate a checkpoint's `quantization_config`; return (quant_method, the engine's fp8_scales it loads into, the name
    suffix of a linear layer's scale tensor)."""
    method = str(qc.get("quant_method", "")).lower()
    if method == "fbgemm_fp8":
        return method, "row", "weight_scale"
    if method != "fp8":
        raise ValueError(f"quant_method {method!r}: only 'fbgemm_fp8' and 'fp8' checkpoints are supported")
    fmt = str(qc.get("fmt", "e4m3")).lower()
    if fmt != "e4m3":
        raise ValueError(f"fp8 checkpoint with fmt={fmt!r}: only e4m3 weights are supported")
    block = qc.get("weight_block_size")
    if block is None:
        return method, "row", "weight_scale_inv"               # one scale per tensor: the row format, scalar repeated
    if list(block) != [F8.BLOCK, F8.BLOCK]:
        raise ValueError(f"fp8 checkpoint with weight_block_size={list(block)}: only [{F8.BLOCK}, {F8.BLOCK}] blocks are supported")
    return method, "block128", "weight_scale_inv"


def _t8(q: torch.Tensor) -> torch.Tensor:
    """The transpose of an e4m3 matrix, contiguous (the codes are moved, not converted)."""
    return q.view(torch.uint8).t().contiguous().view(torch.float8_e4m3fn)


def load_fp8_checkpoint(engine: MoEEngine, shards: Union[str, Sequence[str]], quantization_config: dict, model_type: str,
                        resident: bool = True) -> List[int]:
    """Load the routed experts, router weights and shared experts of a published FP8 checkpoint (its safetensors `shards`,
    its config's `quantization_config`, `model_type` "mixtral", "qwen2_moe" / "qwen3_moe", "deepseek_v3" or "llama4") into
    `engine`, an fp8 engine (`MoEEngine(dtype=torch.bfloat16, expert_dtype=torch.float8_e4m3fn, fp8_scales=...)`), without
    changing a weight byte.  Tensors are read one at a time with `safetensors.safe_open`.

    quant_method "fbgemm_fp8" (Llama 4 Maverick FP8, transformers' fbgemm quantiser): one fp32 scale per output channel,
    loaded into an engine with fp8_scales="row".  Llama 4 stores a layer's experts fused and transposed:
    feed_forward.experts.gate_up_proj e4m3 [E, H, 2I] with gate_up_proj_scale [E, 1, 2I] and down_proj [E, I, H] with
    down_proj_scale [E, H, 1]; the router is feed_forward.router.weight; layers live under model.layers or
    language_model.model.layers, and the MoE layers are the ones with a router.  Other models store one linear layer per
    matrix: weight e4m3 [out, in] with weight_scale [out, 1].
    quant_method "fp8" (transformers' fine-grained FP8): weight e4m3 with weight_scale_inv, which multiplies.  With
    weight_block_size [128, 128] (DeepSeek-V3 / R1, Qwen3-MoE FP8) the scale is a [out/128, in/128] grid, loaded into a
    block engine (fp8_scales="block128"); without a block size it is one scalar per tensor, loaded into a row engine with
    the scalar repeated over the rows.
    Names otherwise as `load_int4_checkpoint`: Mixtral model.layers.{l}.block_sparse_moe.experts.{e}.w{1,2,3} and
    ...block_sparse_moe.gate.weight; DeepSeek / Qwen model.layers.{l}.mlp.experts.{e}.{gate,up,down}_proj, mlp.gate.weight
    (layers without it are skipped), mlp.gate.e_score_correction_bias for a V3 router, and the Qwen shared-expert gate
    mlp.shared_expert_gate.weight.  Shared experts (mlp.shared_experts, mlp.shared_expert, feed_forward.shared_expert) may
    be stored plain or in FP8; either way they are registered dequantised to bf16.  `resident=False` registers the routed
    experts as pinned host blobs (offload).
    The engine then computes the bf16 layer on the dequantised weights (`fp8.dequantize_row` / `dequantize_block128`), not
    the checkpoint's own forward with FP8 activations.
    Refused with a message: other methods, formats or block sizes, a checkpoint whose scale layout does not match the
    engine's fp8_scales, a model type that does not match the engine's expert type or router, dimensions that are not
    multiples of 128, tensors of the wrong dtype or shape, and a missing tensor.  Returns the layers it loaded."""
    from safetensors import safe_open

    method, fmt, scale_name = _fp8_layout(quantization_config)
    if not engine.fp8 or engine.dtype != torch.bfloat16:
        raise ValueError("load_fp8_checkpoint needs an fp8 engine with bf16 activations "
                         "(MoEEngine(dtype=torch.bfloat16, expert_dtype=torch.float8_e4m3fn))")
    if engine.fp8_scales != fmt:
        raise ValueError(f"this {method} checkpoint holds {'per-row' if fmt == 'row' else '128x128 block'} scales: it loads "
                         f"into an engine with fp8_scales={fmt!r}, not {engine.fp8_scales!r}")
    mixtral = model_type == "mixtral"
    qwen = model_type in ("qwen2_moe", "qwen3_moe")
    llama4 = model_type == "llama4"
    if not (mixtral or qwen or llama4 or model_type.startswith("deepseek")):
        raise ValueError(f"model_type {model_type!r}: Mixtral, Qwen-MoE, DeepSeek and Llama 4 checkpoints are supported")
    if llama4 and method != "fbgemm_fp8":
        raise ValueError(f"a Llama 4 checkpoint with quant_method {method!r}: only fbgemm_fp8 Llama 4 experts are supported")
    if mixtral != (engine.expert_type == L.EXPERT_MIXTRAL):
        raise ValueError(f"model_type {model_type!r} does not match the engine's expert_type {engine.expert_type}")
    if qwen != (engine.router == L.ROUTER_QWEN_MOE) or llama4 != (engine.router == L.ROUTER_LLAMA4):
        raise ValueError(f"model_type {model_type!r} does not match the engine's router {engine.router}")
    H, I, E, Is = engine.H, engine.I, engine.E, engine.shared_inter
    if H % F8.BLOCK or I % F8.BLOCK:
        raise ValueError(f"hidden {H} and inter {I} must be multiples of {F8.BLOCK} for fp8 experts")
    if isinstance(shards, str):
        shards = [shards]
    e4m3 = torch.float8_e4m3fn
    with contextlib.ExitStack() as stack:
        files = [stack.enter_context(safe_open(path, framework="pt", device="cpu")) for path in shards]
        where: Dict[str, object] = {k: f for f in files for k in f.keys()}

        def get(key: str) -> torch.Tensor:
            return where[key].get_tensor(key)

        def scales_of(key: str, s: torch.Tensor, rows: int, cols: int) -> torch.Tensor:
            """The engine's scales of a [rows, cols] matrix from its checkpoint scale tensor `key` (fp32 values kept)."""
            if s.dtype not in (torch.float32, torch.bfloat16, torch.float16):
                raise ValueError(f"{key}: scales must be floating point, got {s.dtype}")
            s = s.float()                                          # (exact from bf16 / fp16)
            if fmt == "block128":
                if tuple(s.shape) != (rows // F8.BLOCK, cols // F8.BLOCK):
                    raise ValueError(f"{key}: shape {tuple(s.shape)} is not the 128x128 block grid of a [{rows}, {cols}] matrix")
                return s.contiguous()
            if method == "fp8":                                    # per-tensor: one scalar
                if s.numel() != 1:
                    raise ValueError(f"{key}: shape {tuple(s.shape)} is not the single scale of a per-tensor checkpoint")
                return s.reshape(1).expand(rows).contiguous()
            if tuple(s.shape) not in ((rows,), (rows, 1)):
                raise ValueError(f"{key}: shape {tuple(s.shape)} is not one scale per row of a [{rows}, {cols}] matrix")
            return s.reshape(rows).contiguous()

        def codes(key: str, q: torch.Tensor, shape) -> torch.Tensor:
            if q.dtype != e4m3 or tuple(q.shape) != tuple(shape):
                raise ValueError(f"{key}: expected float8_e4m3fn {tuple(shape)}, got {q.dtype} {tuple(q.shape)}")
            return q

        def linear(prefix: str, rows: int, cols: int):
            """(q, s) of one per-matrix FP8 linear layer."""
            q = codes(f"{prefix}.weight", get(f"{prefix}.weight"), (rows, cols))
            key = f"{prefix}.{scale_name}"
            return q, scales_of(key, get(key), rows, cols)

        def dequantize(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
            return F8.dequantize_row(q, s) if fmt == "row" else F8.dequantize_block128(q, s)

        def shared(prefix: str, rows: int, cols: int) -> torch.Tensor:
            """A shared expert's linear layer in bf16: stored plain, or FP8 dequantised."""
            w = get(f"{prefix}.weight")
            if tuple(w.shape) != (rows, cols):
                raise ValueError(f"{prefix}.weight: expected shape {(rows, cols)}, got {tuple(w.shape)}")
            if w.dtype != e4m3:
                return w.to(engine.dtype)
            key = f"{prefix}.{scale_name}"
            if key not in where:
                raise ValueError(f"the checkpoint has no tensor {key} (the scale of the FP8 {prefix}.weight)")
            return dequantize(w, scales_of(key, get(key), rows, cols))

        if llama4:
            root = next((r for r in ("model.layers", "language_model.model.layers")
                         if any(f"{r}.{l}.feed_forward.router.weight" in where for l in range(engine.L))), None)
            if root is None:
                raise ValueError("the checkpoint has no Llama 4 MoE layer (no {model.,language_model.model.}layers.*"
                                 ".feed_forward.router.weight)")
            layers = [l for l in range(engine.L) if f"{root}.{l}.feed_forward.router.weight" in where]
            moe, router, shared_name = "feed_forward", "router", "shared_expert"
            names = ("gate_proj", "up_proj", "down_proj")
        elif mixtral:
            root, moe, router, shared_name = "model.layers", "block_sparse_moe", "gate", None
            layers = list(range(engine.L))
            names = ("w1", "w2", "w3")                                 # reference order: w1 | w2 | w3
        else:
            root, moe, router = "model.layers", "mlp", "gate"
            shared_name = "shared_expert" if qwen else "shared_experts"
            layers = [l for l in range(engine.L) if f"{root}.{l}.mlp.gate.weight" in where]
            names = ("gate_proj", "up_proj", "down_proj")              # DeepSeek order: gate | up | down
        shapes = {"w1": (I, H), "w2": (H, I), "w3": (I, H), "gate_proj": (I, H), "up_proj": (I, H), "down_proj": (H, I)}
        shared_shapes = {"gate_proj": (Is, H), "up_proj": (Is, H), "down_proj": (H, Is)}
        need = []
        for l in layers:
            base = f"{root}.{l}.{moe}"
            need.append(f"{base}.{router}.weight")
            if llama4:
                need += [f"{base}.experts.{n}{p}" for n in ("gate_up_proj", "down_proj") for p in ("", "_scale")]
            else:
                need += [f"{base}.experts.{e}.{n}.{p}" for e in range(E) for n in names for p in ("weight", scale_name)]
            if shared_name and Is > 0:
                need += [f"{base}.{shared_name}.{n}.weight" for n in names]
            if qwen and Is > 0:
                need.append(f"{base}.shared_expert_gate.weight")
            if engine.router == L.ROUTER_DEEPSEEK_V3:
                need.append(f"{base}.gate.e_score_correction_bias")
        missing = [k for k in need if k not in where]
        if missing:
            raise ValueError(f"the checkpoint has no tensor {missing[0]} ({len(missing)} missing)")
        for l in layers:
            base = f"{root}.{l}.{moe}"
            if llama4:
                # Llama4TextExperts computes x @ gate_up_proj[e]: column j of [H, 2I] is output channel j, scaled by
                # gate_up_proj_scale[e, 0, j]; the engine takes the nn.Linear [out, in] transposes
                k_gu, k_dn = f"{base}.experts.gate_up_proj", f"{base}.experts.down_proj"
                gu, dn = codes(k_gu, get(k_gu), (E, H, 2 * I)), codes(k_dn, get(k_dn), (E, I, H))
                gus, dns = get(f"{k_gu}_scale"), get(f"{k_dn}_scale")
                if tuple(gus.shape) != (E, 1, 2 * I) or tuple(dns.shape) != (E, H, 1):
                    raise ValueError(f"{k_gu}_scale / {k_dn}_scale: shapes {tuple(gus.shape)} / {tuple(dns.shape)} are not "
                                     f"per-output-channel scales {(E, 1, 2 * I)} / {(E, H, 1)}")

                def expert(e):
                    return [(_t8(gu[e][:, :I]), scales_of(f"{k_gu}_scale", gus[e, 0, :I], I, H)),
                            (_t8(gu[e][:, I:]), scales_of(f"{k_gu}_scale", gus[e, 0, I:], I, H)),
                            (_t8(dn[e]), scales_of(f"{k_dn}_scale", dns[e, :, 0], H, I))]
            else:
                def expert(e):
                    return [linear(f"{base}.experts.{e}.{n}", *shapes[n]) for n in names]
            for e in range(E):
                qs, ss = zip(*expert(e))
                if resident:
                    engine.load_expert(l, e, qs, scales=ss)
                else:
                    engine.register_expert(l, e, qs, scales=ss)
            if shared_name and Is > 0:
                engine.register_shared(l, [shared(f"{base}.{shared_name}.{n}", *shared_shapes[n]) for n in names])
            if qwen and Is > 0:
                engine.set_shared_gate(l, get(f"{base}.shared_expert_gate.weight").to(engine.dtype))
            engine.set_gate(l, get(f"{base}.{router}.weight"))
            if engine.router == L.ROUTER_DEEPSEEK_V3:
                engine.set_gate_bias(l, get(f"{base}.gate.e_score_correction_bias").float())
    return layers
