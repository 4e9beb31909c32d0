"""CPU: the Qwen2-MoE / Qwen3-MoE router (B2M_ROUTER_QWEN_MOE) through the C-ABI layer on the host simulation of
tests/test_host_sim.py (api.cu compiled unchanged against stand-in launchers): the configurations b2m_ctx_create_ex
accepts and refuses, the argument checks of b2m_set_shared_gate, the missing-gate state error, the expert-parallel
refusal, the shared-gate phase of the combine (launched ahead of the shared GEMMs, counted in kernel_launches) and the new workspaces.  Then
hf.load_int4_checkpoint on synthetic Qwen2-MoE / Qwen3-MoE AWQ and GPTQ shards, checked against a recording engine."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import int4_checkpoint_packers as P  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from moe_infinity_b200 import hf  # noqa: E402
from moe_infinity_b200.int4 import dequantize_g128  # noqa: E402
from test_host_sim import Ctx, _SO, sim, take_log  # noqa: E402,F401  (sim: the module-scoped library fixture)

needs_sim = pytest.mark.skipif(_SO is None, reason="nvcc / g++ not available to build the host simulation")


def _qwen(lib, **kw):
    kw.setdefault("n_group", 1)
    kw.setdefault("topk_group", 1)
    kw.setdefault("expert_type", L.EXPERT_DEEPSEEK)
    return Ctx(lib, router=L.ROUTER_QWEN_MOE, **kw)


@needs_sim
def test_qwen_router_is_accepted_on_cpu(sim):
    for kw in (dict(E=60, k=4, shared_inter=256), dict(E=128, k=8, norm_topk_prob=1), dict(E=16, k=1, norm_topk_prob=1),
               dict(E=8, k=2, dtype=L.DTYPE_F16, gate_dtype=L.DTYPE_F16, shared_inter=128)):
        c = _qwen(sim, **kw)
        assert c.rc == 0, (kw, c.err())
        c.close()


@needs_sim
@pytest.mark.parametrize("kw,what", [
    (dict(expert_type=L.EXPERT_MIXTRAL), "expert_type"), (dict(dtype=L.DTYPE_F32), "bf16 or f16"),
    (dict(n_group=2, topk_group=1), "n_group"), (dict(n_group=1, topk_group=2), "topk_group"),
    (dict(n_group=0, topk_group=0), "n_group"), (dict(routed_scaling_factor=2.5), "routed_scaling_factor")])
def test_qwen_router_refuses_other_configs_on_cpu(sim, kw, what):
    c = _qwen(sim, **kw)
    assert c.rc == L.B2M_EINVAL, kw
    msg = (sim.b2m_last_error(None) or b"").decode()
    assert "qwen_moe" in msg and what in msg, msg


@needs_sim
def test_set_shared_gate_arguments_on_cpu(sim):
    c = _qwen(sim, shared_inter=128)
    assert c.rc == 0, c.err()
    w = np.zeros(c.H, dtype=np.uint16)
    assert sim.b2m_set_shared_gate(c.h, -1, w.ctypes.data) == L.B2M_EINVAL
    assert sim.b2m_set_shared_gate(c.h, c.L, w.ctypes.data) == L.B2M_EINVAL and "out of range" in c.err()
    assert sim.b2m_set_shared_gate(c.h, 0, None) == L.B2M_EINVAL and "null" in c.err()
    assert sim.b2m_set_shared_gate(c.h, 0, w.ctypes.data) == 0, c.err()
    c.close()
    c = _qwen(sim)                                   # Qwen3: no shared experts, no gate
    assert c.rc == 0, c.err()
    assert sim.b2m_set_shared_gate(c.h, 0, w.ctypes.data) == L.B2M_EINVAL and "no shared experts" in c.err()
    c.close()
    for router, extra in ((L.ROUTER_MIXTRAL, {}), (L.ROUTER_DEEPSEEK_GREEDY, {}), (L.ROUTER_DEEPSEEK_V3, dict(n_group=4, topk_group=2))):
        m = Ctx(sim, router=router, expert_type=L.EXPERT_DEEPSEEK, shared_inter=128, **extra)
        assert m.rc == 0, m.err()
        assert sim.b2m_set_shared_gate(m.h, 0, w.ctypes.data) == L.B2M_EINVAL and "qwen_moe" in m.err(), m.err()
        m.close()


GATE_LINE = "combine T={T} mode=5 shared=0 ep_collect=0 dtype=0"     # the stand-in launcher's record of the gate phase


def _register_shared(c, layer):
    blob = np.zeros(3 * c.H * 128 * 2, dtype=np.uint8)
    c.blobs[("shared", layer)] = blob
    assert c.lib.b2m_register_shared(c.h, layer, blob.ctypes.data, blob.nbytes) == 0, c.err()


@needs_sim
def test_missing_shared_gate_is_a_state_error_on_cpu(sim):
    c = _qwen(sim, shared_inter=128, num_slots=3 * 8)
    assert c.rc == 0, c.err()
    c.register_all()
    for l in range(c.L):
        _register_shared(c, l)
    T = 5
    lg = np.random.default_rng(0).standard_normal((T, c.E)).astype(np.float32)
    x = np.zeros((T, c.H), dtype=np.uint16)
    out = np.zeros((T, c.H), dtype=np.uint16)
    assert c.forward(0, lg) == L.B2M_ESTATE
    assert "layer 0 has no shared-expert gate" in c.err(), c.err()
    assert sim.b2m_route(c.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == 0, c.err()
    assert sim.b2m_run_experts(c.h, 0, T, None) == 0, c.err()
    assert sim.b2m_combine(c.h, 0, x.ctypes.data, T, out.ctypes.data, None) == L.B2M_ESTATE
    w = np.zeros(c.H, dtype=np.uint16)
    assert sim.b2m_set_shared_gate(c.h, 0, w.ctypes.data) == 0
    take_log(sim)
    s0 = c.stats()["kernel_launches"]
    assert c.forward(0, lg) == 0, c.err()
    log = take_log(sim)
    # the gate phase of the combine (mode 5, COMBINE_QWEN_GATE) runs first on the shared-expert stream, ahead of the shared
    # GEMMs; the combine proper (mode 4, COMBINE_QWEN) follows the routed experts
    assert log[0] == GATE_LINE.format(T=5), log
    assert log[1].startswith("gemm") and "single_n=5" in log[1], log
    comb = [ln for ln in log if ln.startswith("combine")]
    assert comb == [GATE_LINE.format(T=5), "combine T=5 mode=4 shared=1 ep_collect=0 dtype=0"], comb
    n_qwen = c.stats()["kernel_launches"] - s0
    assert c.forward(1, lg) == L.B2M_ESTATE                      # the gate is per layer
    c.close()
    # the same forward with an ungated shared expert (DeepSeek combine) launches exactly one kernel less
    d = Ctx(sim, router=L.ROUTER_DEEPSEEK_GREEDY, expert_type=L.EXPERT_DEEPSEEK, shared_inter=128, num_slots=3 * 8)
    assert d.rc == 0, d.err()
    d.register_all()
    _register_shared(d, 0)
    d.forward(0, lg)                                             # the first forward of a layer also uploads its slot table
    take_log(sim)
    s0 = d.stats()["kernel_launches"]
    assert d.forward(0, lg) == 0, d.err()
    assert not any("mode=5" in ln for ln in take_log(sim))
    assert n_qwen == d.stats()["kernel_launches"] - s0 + 1
    d.close()


@needs_sim
def test_qwen3_combine_mode_and_numerics_on_cpu(sim):
    for numerics, mode in ((L.NUMERICS_REFERENCE, 4), (L.NUMERICS_FP32, 3)):
        c = _qwen(sim, num_slots=3 * 8, numerics=numerics)
        assert c.rc == 0, c.err()
        c.register_all()
        take_log(sim)
        assert c.forward(0, np.random.default_rng(1).standard_normal((3, c.E)).astype(np.float32)) == 0, c.err()
        log = take_log(sim)
        assert not any("mode=5" in ln for ln in log)
        assert [ln for ln in log if ln.startswith("combine")] == [f"combine T=3 mode={mode} shared=0 ep_collect=0 dtype=0"]
        c.close()


@needs_sim
def test_qwen_workspaces_on_cpu(sim):
    p = C.c_void_p()
    c = _qwen(sim, shared_inter=128)
    assert sim.b2m_ws_ptr(c.h, L.WS["shared_gate"], C.byref(p)) == 0 and p.value
    assert sim.b2m_ws_ptr(c.h, L.WS["y_shared"], C.byref(p)) == 0 and p.value
    c.close()
    c = _qwen(sim)
    assert sim.b2m_ws_ptr(c.h, L.WS["shared_gate"], C.byref(p)) == L.B2M_ESTATE
    assert sim.b2m_ws_ptr(c.h, L.WS["y_shared"], C.byref(p)) == L.B2M_ESTATE
    c.close()
    c = Ctx(sim, router=L.ROUTER_DEEPSEEK_GREEDY, expert_type=L.EXPERT_DEEPSEEK, shared_inter=128)
    assert sim.b2m_ws_ptr(c.h, L.WS["shared_gate"], C.byref(p)) == L.B2M_ESTATE
    assert sim.b2m_ws_ptr(c.h, L.WS["y_shared"], C.byref(p)) == 0 and p.value
    c.close()


@needs_sim
def test_expert_parallel_is_refused_on_cpu(sim):
    c = _qwen(sim, max_tokens=64)
    assert c.rc == 0, c.err()
    send = np.zeros((2, 8, c.H), dtype=np.uint16)
    cnt = np.zeros(c.E, dtype=np.int32)
    assert sim.b2m_ep_pack(c.h, 2, 0, 8, 4, send.ctypes.data, cnt.ctypes.data, None) == L.B2M_EUNSUPPORTED
    assert "qwen_moe" in c.err(), c.err()
    handle = (C.c_uint8 * 64)()
    assert sim.b2m_ep_p2p_init(c.h, 2, 0, 8, handle) == L.B2M_EUNSUPPORTED
    c.close()


# ---------------------------------------------------------------- hf.load_int4_checkpoint, Qwen model types
class _FakeEngine:
    """Records what load_int4_checkpoint hands an engine (the real one needs a GPU)."""

    def __init__(self, L_, E, H, I, shared_inter=0, router=L.ROUTER_QWEN_MOE):
        self.int4, self.dtype = True, torch.float16
        self.L, self.E, self.H, self.I = L_, E, H, I
        self.expert_type, self.shared_inter, self.router = L.EXPERT_DEEPSEEK, shared_inter, router
        self.experts, self.shared, self.gates, self.shared_gates = {}, {}, {}, {}

    def load_expert(self, l, e, qs, scales=None, zeros=None):
        self.experts[(l, e)] = (qs, scales, zeros)

    register_expert = load_expert

    def register_shared(self, l, ws):
        self.shared[l] = ws

    def set_gate(self, l, w):
        self.gates[l] = w

    def set_shared_gate(self, l, w):
        self.shared_gates[l] = w


def _put(tensors, truth, name, out, n_in, g, method):
    q, s, z = P.random_qsz(out, n_in, g, z_lo=0 if method == "awq" else 1)   # (GPTQ v1 stores z - 1)
    truth[name] = P.fp16_dequant(q, s, z)
    if method == "awq":
        qw, qz, sc = P.awq_pack(q, s, z)
    else:
        qw, qz, sc, gi = P.gptq_pack(q, s, z)
        tensors[f"{name}.g_idx"] = gi
    tensors[f"{name}.qweight"], tensors[f"{name}.qzeros"], tensors[f"{name}.scales"] = qw, qz, sc


def _qwen_shards(method, shared, L_=3, E=4, H=256, I=128, Is=256, seed=80, gate_form="plain"):
    """Layer 0 dense (mlp_only_layers), layers 1.. sparse."""
    g = torch.Generator().manual_seed(seed)
    tensors, truth = {"model.layers.0.mlp.gate_proj.weight": torch.zeros(4, 4, dtype=torch.float16)}, {}
    for l in range(1, L_):
        base = f"model.layers.{l}.mlp"
        tensors[f"{base}.gate.weight"] = torch.randn(E, H, generator=g).to(torch.float16)
        for e in range(E):
            for n, (o, i) in (("gate_proj", (I, H)), ("up_proj", (I, H)), ("down_proj", (H, I))):
                _put(tensors, truth, f"{base}.experts.{e}.{n}", o, i, g, method)
        if shared:
            for n, (o, i) in (("gate_proj", (Is, H)), ("up_proj", (Is, H)), ("down_proj", (H, Is))):
                _put(tensors, truth, f"{base}.shared_expert.{n}", o, i, g, method)
            if gate_form == "plain":
                tensors[f"{base}.shared_expert_gate.weight"] = torch.randn(1, H, generator=g).to(torch.float16)
            elif gate_form == "quantised":
                tensors[f"{base}.shared_expert_gate.qweight"] = torch.zeros(H // 8, 1, dtype=torch.int32)
    return tensors, truth


AWQ_CFG = dict(quant_method="awq", bits=4, group_size=128, zero_point=True, version="gemm")
GPTQ_CFG = dict(quant_method="gptq", bits=4, group_size=128, desc_act=False)


@pytest.mark.parametrize("method,model_type,shared", [("awq", "qwen2_moe", True), ("gptq", "qwen2_moe", True),
                                                      ("gptq", "qwen3_moe", False), ("awq", "qwen3_moe", False)])
def test_load_qwen_int4_checkpoint(tmp_path, method, model_type, shared):
    H, I, Is, E = 256, 128, 256, 4
    tensors, truth = _qwen_shards(method, shared, E=E, H=H, I=I, Is=Is)
    eng = _FakeEngine(3, E, H, I, shared_inter=Is if shared else 0)
    cfg = AWQ_CFG if method == "awq" else GPTQ_CFG
    assert hf.load_int4_checkpoint(eng, P.write_shards(str(tmp_path), tensors), cfg, model_type) == [1, 2]
    for l in (1, 2):
        base = f"model.layers.{l}.mlp"
        for e in range(E):
            qs, ss, zs = eng.experts[(l, e)]
            for n, q, s_, z in zip(("gate_proj", "up_proj", "down_proj"), qs, ss, zs):
                w = dequantize_g128(q, s_, z, torch.float16)
                assert torch.equal(w.view(torch.int16), truth[f"{base}.experts.{e}.{n}"].view(torch.int16)), (l, e, n)
        assert torch.equal(eng.gates[l], tensors[f"{base}.gate.weight"])
        if shared:
            for n, w in zip(("gate_proj", "up_proj", "down_proj"), eng.shared[l]):
                assert w.dtype == torch.float16 and torch.equal(w.view(torch.int16),
                                                                 truth[f"{base}.shared_expert.{n}"].view(torch.int16))
            sg = eng.shared_gates[l]
            assert sg.dtype == torch.float16 and torch.equal(sg, tensors[f"{base}.shared_expert_gate.weight"])
        else:
            assert not eng.shared and not eng.shared_gates


@pytest.mark.parametrize("gate_form,match", [("missing", "shared_expert_gate.weight"),
                                             ("quantised", "stores model.layers.1.mlp.shared_expert_gate quantised")])
def test_load_qwen_refuses_shared_gate(tmp_path, gate_form, match):
    tensors, _ = _qwen_shards("gptq", True, E=2, gate_form=gate_form)
    eng = _FakeEngine(3, 2, 256, 128, shared_inter=256)
    with pytest.raises(ValueError, match=match):
        hf.load_int4_checkpoint(eng, P.write_shards(str(tmp_path), tensors), GPTQ_CFG, "qwen2_moe")


def test_load_qwen_refuses_other_router(tmp_path):
    tensors, _ = _qwen_shards("gptq", False, E=2)
    shards = P.write_shards(str(tmp_path), tensors)
    with pytest.raises(ValueError, match="does not match the engine's router"):
        hf.load_int4_checkpoint(_FakeEngine(3, 2, 256, 128, router=L.ROUTER_DEEPSEEK_GREEDY), shards, GPTQ_CFG, "qwen3_moe")
