"""CPU: hf.load_fp8_checkpoint on synthetic safetensors shards, one per published FP8 layout, into a stand-in engine that
records every call.

* fbgemm_fp8 fused Llama 4 experts (under language_model.model.layers with a plain bf16 shared expert, under model.layers
  with an FbgemmFp8Linear shared expert; a dense layer without a router between MoE layers);
* fbgemm_fp8 per-Linear experts (Mixtral, Qwen2-MoE with its shared expert and shared-expert gate);
* fine-grained fp8 with 128x128 blocks (DeepSeek-V3 with correction bias and an FP8 shared expert, Qwen3-MoE);
* fine-grained fp8 with one scale per tensor (Mixtral).
Checked: the e4m3 bytes and fp32 scales handed to the engine (row scales for fbgemm and per-tensor, block grids for the
block layout), the dequantised bf16 shared experts, the router, correction-bias and shared-gate calls, resident and host-backed
loading, and each refusal."""
from __future__ import annotations

from typing import Dict

import pytest
import torch

from int4_checkpoint_packers import write_shards
from moe_infinity_b200 import _lib as L
from moe_infinity_b200 import hf
from moe_infinity_b200.fp8 import dequantize_block128, dequantize_row

FP8 = torch.float8_e4m3fn
BF16 = torch.bfloat16
H, I, E, SI = 256, 128, 4, 256


class _Engine:
    """Records what the loader hands to an fp8 MoEEngine."""

    def __init__(self, scales="row", expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, shared_inter=0,
                 layers=2, H=H, I=I):
        self.fp8, self.dtype, self.fp8_scales = True, BF16, scales
        self.expert_type, self.router, self.shared_inter = expert_type, router, shared_inter
        self.L, self.E, self.H, self.I = layers, E, H, I
        self.experts, self.shared, self.gates, self.biases, self.shared_gates = {}, {}, {}, {}, {}
        self.how = set()

    def load_expert(self, l, e, qs, scales=None):
        self.experts[(l, e)] = (qs, scales)
        self.how.add("resident")

    def register_expert(self, l, e, qs, scales=None):
        self.experts[(l, e)] = (qs, scales)
        self.how.add("host")

    def register_shared(self, l, ws):
        self.shared[l] = ws

    def set_gate(self, l, w):
        self.gates[l] = w

    def set_gate_bias(self, l, b):
        self.biases[l] = b

    def set_shared_gate(self, l, w):
        self.shared_gates[l] = w


def _codes(g, *shape):
    c = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    c[(c & 0x7f) == 0x7f] = 0x38                                  # no NaN codes
    return c.view(FP8)


def _scales(g, *shape):
    return torch.rand(shape, generator=g) * 0.01 + 1e-4


def _same8(a, b):
    return a.dtype == FP8 and b.dtype == FP8 and a.shape == b.shape and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ------------------------------------------------------------------------------------------------ Llama 4, fused fbgemm
def _llama4_ckpt(g, root, fp8_shared, moe_layers=(1, 3)):
    t: Dict[str, torch.Tensor] = {}
    want = {}
    for l in moe_layers:
        b = f"{root}.{l}.feed_forward"
        gu, dn = _codes(g, E, H, 2 * I), _codes(g, E, I, H)
        gus, dns = _scales(g, E, 1, 2 * I), _scales(g, E, H, 1)
        t.update({f"{b}.experts.gate_up_proj": gu, f"{b}.experts.gate_up_proj_scale": gus,
                  f"{b}.experts.down_proj": dn, f"{b}.experts.down_proj_scale": dns,
                  f"{b}.router.weight": torch.randn(E, H, generator=g).to(BF16)})
        want[l] = [((gu[e][:, :I].t(), gus[e, 0, :I]), (gu[e][:, I:].t(), gus[e, 0, I:]), (dn[e].t(), dns[e, :, 0]))
                   for e in range(E)]
        sh = []
        for n, (r, c) in (("gate_proj", (I, H)), ("up_proj", (I, H)), ("down_proj", (H, I))):
            if fp8_shared:
                q, s = _codes(g, r, c), _scales(g, r, 1)
                t[f"{b}.shared_expert.{n}.weight"], t[f"{b}.shared_expert.{n}.weight_scale"] = q, s
                sh.append(dequantize_row(q, s))
            else:
                w = torch.randn(r, c, generator=g).to(BF16)
                t[f"{b}.shared_expert.{n}.weight"] = w
                sh.append(w)
        want[(l, "shared")] = sh
    t[f"{root}.2.feed_forward.gate_proj.weight"] = torch.randn(16, H, generator=g).to(BF16)   # a dense layer
    return t, want


@pytest.mark.parametrize("root,fp8_shared,resident", [("language_model.model.layers", False, True),
                                                       ("model.layers", True, False)])
def test_llama4_fbgemm(tmp_path, root, fp8_shared, resident):
    g = torch.Generator().manual_seed(1)
    t, want = _llama4_ckpt(g, root, fp8_shared)
    paths = write_shards(str(tmp_path), t, nshards=3)
    eng = _Engine("row", router=L.ROUTER_LLAMA4, shared_inter=I, layers=4)
    layers = hf.load_fp8_checkpoint(eng, paths, {"quant_method": "fbgemm_fp8"}, "llama4", resident=resident)
    assert layers == [1, 3]
    assert eng.how == {"resident" if resident else "host"}
    assert sorted(eng.experts) == [(l, e) for l in (1, 3) for e in range(E)]
    for l in (1, 3):
        for e in range(E):
            qs, ss = eng.experts[(l, e)]
            for (q, s), (wq, ws) in zip(zip(qs, ss), want[l][e]):
                assert _same8(q, wq) and q.is_contiguous()
                assert s.dtype == torch.float32 and torch.equal(s, ws)
        for got, w in zip(eng.shared[l], want[(l, "shared")]):
            assert got.dtype == BF16 and torch.equal(got, w)
        assert torch.equal(eng.gates[l], t[f"{root}.{l}.feed_forward.router.weight"])
    assert not eng.biases and not eng.shared_gates


# ------------------------------------------------------------------------------------------------ per-Linear layouts
def _linear_ckpt(g, model, layout, layers=(0, 1)):
    """(tensors, want): per-matrix FP8 linear layers; layout "fbgemm" ([out, 1] scales), "block" ([out/128, in/128]
    weight_scale_inv) or "tensor" (one weight_scale_inv scalar)."""
    mixtral = model == "mixtral"
    names = (("w1", (I, H)), ("w2", (H, I)), ("w3", (I, H))) if mixtral else \
        (("gate_proj", (I, H)), ("up_proj", (I, H)), ("down_proj", (H, I)))
    moe = "block_sparse_moe" if mixtral else "mlp"
    sname = "weight_scale" if layout == "fbgemm" else "weight_scale_inv"

    def quant(r, c):
        q = _codes(g, r, c)
        if layout == "fbgemm":
            s = _scales(g, r, 1)
            return q, s, s.reshape(r), dequantize_row(q, s)
        if layout == "tensor":
            s = _scales(g)
            return q, s, s.expand(r).contiguous(), dequantize_row(q, s.expand(r).contiguous())
        s = _scales(g, r // 128, c // 128)
        return q, s, s, dequantize_block128(q, s)

    t, want = {}, {}
    for l in layers:
        b = f"model.layers.{l}.{moe}"
        t[f"{b}.gate.weight"] = torch.randn(E, H, generator=g).to(BF16 if model != "deepseek_v3" else torch.float32)
        for e in range(E):
            want[(l, e)] = []
            for n, (r, c) in names:
                q, s, s_eng, _ = quant(r, c)
                t[f"{b}.experts.{e}.{n}.weight"], t[f"{b}.experts.{e}.{n}.{sname}"] = q, s
                want[(l, e)].append((q, s_eng))
        shared = {"qwen2_moe": "shared_expert", "deepseek_v3": "shared_experts"}.get(model)
        if shared:
            want[(l, "shared")] = []
            for n, (r, c) in names:
                r, c = (SI, H) if n != "down_proj" else (H, SI)
                q, s, _, w = quant(r, c)
                t[f"{b}.{shared}.{n}.weight"], t[f"{b}.{shared}.{n}.{sname}"] = q, s
                want[(l, "shared")].append(w)
        if model == "qwen2_moe":
            t[f"{b}.shared_expert_gate.weight"] = torch.randn(1, H, generator=g).to(BF16)
        if model == "deepseek_v3":
            t[f"{b}.gate.e_score_correction_bias"] = torch.randn(E, generator=g)
    return t, want


CASES = {   # name: (model, layout, quantization_config, engine kwargs)
    "mixtral_fbgemm": ("mixtral", "fbgemm", {"quant_method": "fbgemm_fp8"},
                       dict(scales="row", expert_type=L.EXPERT_MIXTRAL, router=L.ROUTER_MIXTRAL)),
    "qwen2_moe_fbgemm": ("qwen2_moe", "fbgemm", {"quant_method": "fbgemm_fp8"},
                         dict(scales="row", router=L.ROUTER_QWEN_MOE, shared_inter=SI)),
    "deepseek_v3_block": ("deepseek_v3", "block", {"quant_method": "fp8", "fmt": "e4m3", "weight_block_size": [128, 128]},
                          dict(scales="block128", router=L.ROUTER_DEEPSEEK_V3, shared_inter=SI)),
    "qwen3_moe_block": ("qwen3_moe", "block", {"quant_method": "fp8", "weight_block_size": [128, 128]},
                        dict(scales="block128", router=L.ROUTER_QWEN_MOE)),
    "mixtral_per_tensor": ("mixtral", "tensor", {"quant_method": "fp8", "activation_scheme": "dynamic"},
                           dict(scales="row", expert_type=L.EXPERT_MIXTRAL, router=L.ROUTER_MIXTRAL)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_per_linear_layouts(tmp_path, name):
    model, layout, qc, kw = CASES[name]
    g = torch.Generator().manual_seed(2)
    t, want = _linear_ckpt(g, model, layout)
    paths = write_shards(str(tmp_path), t)
    eng = _Engine(**kw)
    assert hf.load_fp8_checkpoint(eng, paths, qc, model) == [0, 1]
    moe = "block_sparse_moe" if model == "mixtral" else "mlp"
    for l in (0, 1):
        b = f"model.layers.{l}.{moe}"
        for e in range(E):
            qs, ss = eng.experts[(l, e)]
            for q, s, (wq, ws) in zip(qs, ss, want[(l, e)]):
                assert _same8(q, wq) and s.dtype == torch.float32 and torch.equal(s, ws)
        if (l, "shared") in want:
            for got, w in zip(eng.shared[l], want[(l, "shared")]):
                assert got.dtype == BF16 and torch.equal(got, w)
        else:
            assert l not in eng.shared
        assert torch.equal(eng.gates[l], t[f"{b}.gate.weight"])
        if model == "deepseek_v3":
            assert torch.equal(eng.biases[l], t[f"{b}.gate.e_score_correction_bias"])
        if model == "qwen2_moe":
            assert torch.equal(eng.shared_gates[l], t[f"{b}.shared_expert_gate.weight"])
    assert bool(eng.biases) == (model == "deepseek_v3") and bool(eng.shared_gates) == (model == "qwen2_moe")


def test_refusals(tmp_path):
    g = torch.Generator().manual_seed(3)
    t, _ = _linear_ckpt(g, "deepseek_v3", "block")
    paths = write_shards(str(tmp_path), t)
    block = {"quant_method": "fp8", "weight_block_size": [128, 128]}
    v3 = dict(scales="block128", router=L.ROUTER_DEEPSEEK_V3, shared_inter=SI)

    def refused(match, qc=block, model="deepseek_v3", shards=paths, **kw):
        with pytest.raises(ValueError, match=match):
            hf.load_fp8_checkpoint(_Engine(**{**v3, **kw}), shards, qc, model)

    refused("weight_block_size", {"quant_method": "fp8", "weight_block_size": [64, 64]})
    refused("quant_method", {"quant_method": "awq"})
    refused("fmt", {"quant_method": "fp8", "fmt": "e5m2", "weight_block_size": [128, 128]})
    refused("fp8_scales='block128'", scales="row")                      # block checkpoint, row engine
    refused("fp8_scales='row'", {"quant_method": "fbgemm_fp8"})          # row checkpoint, block engine
    refused("router", model="qwen3_moe")                                 # model type vs the engine's router
    refused("expert_type", model="mixtral")
    refused("model_type", model="gpt2")
    refused("multiples of 128", H=200)
    # the scales of the checkpoint do not match what its config promises (per-tensor config, block grids stored)
    refused("single scale", {"quant_method": "fp8"}, scales="row")
    del t["model.layers.1.mlp.experts.2.up_proj.weight_scale_inv"]
    (tmp_path / "missing").mkdir()
    refused("no tensor model.layers.1.mlp.experts.2.up_proj.weight_scale_inv", shards=write_shards(str(tmp_path / "missing"), t))
    with pytest.raises(ValueError, match="fp8 engine"):
        e = _Engine(**v3)
        e.fp8 = False
        hf.load_fp8_checkpoint(e, paths, block, "deepseek_v3")
    # a Llama 4 checkpoint: routed expert codes of the wrong shape, and a fine-grained Llama 4 checkpoint
    t4, _ = _llama4_ckpt(g, "model.layers", False, moe_layers=(1,))
    (tmp_path / "llama4").mkdir()
    p4 = write_shards(str(tmp_path / "llama4"), t4)
    with pytest.raises(ValueError, match="gate_up_proj"):
        hf.load_fp8_checkpoint(_Engine("row", router=L.ROUTER_LLAMA4, shared_inter=I, layers=4, I=2 * I), p4,
                               {"quant_method": "fbgemm_fp8"}, "llama4")
    with pytest.raises(ValueError, match="fbgemm_fp8"):
        hf.load_fp8_checkpoint(_Engine("row", router=L.ROUTER_LLAMA4, shared_inter=I, layers=4), p4, {"quant_method": "fp8"},
                               "llama4")
    with pytest.raises(ValueError, match="no Llama 4 MoE layer"):
        hf.load_fp8_checkpoint(_Engine("row", router=L.ROUTER_LLAMA4, shared_inter=I, layers=4), paths,
                               {"quant_method": "fbgemm_fp8"}, "llama4")
