"""CPU: the Llama 4 router (B2M_ROUTER_LLAMA4) through the C-ABI layer on the host simulation of tests/test_host_sim.py
(api.cu compiled unchanged against stand-in launchers): the configurations b2m_ctx_create_ex accepts and refuses, the
refusals of scores input, input permutations and expert parallelism, the combine mode of both numerics and the launch
count of a forward.  Then hf.patch_llama4 on a tiny CPU Llama4ForCausalLM, checked against a recording engine."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from moe_infinity_b200 import _lib as L  # noqa: E402
from moe_infinity_b200 import hf  # noqa: E402
from test_host_sim import Ctx, _SO, sim, take_log  # noqa: E402,F401  (sim: the module-scoped library fixture)

needs_sim = pytest.mark.skipif(_SO is None, reason="nvcc / g++ not available to build the host simulation")


def _llama4(lib, **kw):
    kw.setdefault("n_group", 1)
    kw.setdefault("topk_group", 1)
    kw.setdefault("expert_type", L.EXPERT_DEEPSEEK)
    kw.setdefault("shared_inter", 128)
    return Ctx(lib, router=L.ROUTER_LLAMA4, **kw)


def _register_shared(c, layer):
    blob = np.zeros(3 * c.H * 128 * 2, dtype=np.uint8)
    c.blobs[("shared", layer)] = blob
    assert c.lib.b2m_register_shared(c.h, layer, blob.ctypes.data, blob.nbytes) == 0, c.err()


@needs_sim
def test_llama4_router_is_accepted_on_cpu(sim):
    for kw in (dict(E=16, k=1), dict(E=128, k=1), dict(E=16, k=4), dict(E=8, k=8),
               dict(E=16, k=2, dtype=L.DTYPE_F16, gate_dtype=L.DTYPE_F16)):
        c = _llama4(sim, **kw)
        assert c.rc == 0, (kw, c.err())
        c.close()


@needs_sim
@pytest.mark.parametrize("kw,what", [
    (dict(expert_type=L.EXPERT_MIXTRAL), "expert_type"), (dict(dtype=L.DTYPE_F32), "bf16 or f16"),
    (dict(n_group=2, topk_group=1), "n_group"), (dict(n_group=1, topk_group=2), "topk_group"),
    (dict(routed_scaling_factor=2.5), "routed_scaling_factor"), (dict(norm_topk_prob=1), "norm_topk_prob"),
    (dict(shared_inter=0), "shared_inter")])
def test_llama4_router_refuses_other_configs_on_cpu(sim, kw, what):
    c = _llama4(sim, **kw)
    assert c.rc == L.B2M_EINVAL, kw
    msg = (sim.b2m_last_error(None) or b"").decode()
    assert "llama4" in msg and what in msg, msg


@needs_sim
def test_scores_input_and_input_perm_are_refused_on_cpu(sim):
    c = _llama4(sim)
    assert c.rc == 0, c.err()
    T = 4
    x = np.zeros((T, c.H), dtype=np.uint16)
    sc = np.full((T, c.E), 1.0 / c.E, dtype=np.float32)
    assert sim.b2m_route(c.h, 0, x.ctypes.data, sc.ctypes.data, 2, L.DTYPE_F32, T, 0, None) == L.B2M_EUNSUPPORTED
    assert "llama4" in c.err() and "scores" in c.err(), c.err()
    out = np.zeros((T, c.H), dtype=np.uint16)
    assert sim.b2m_moe_forward(c.h, 0, x.ctypes.data, sc.ctypes.data, 2, L.DTYPE_F32, T, 0, out.ctypes.data,
                               None) == L.B2M_EUNSUPPORTED
    perm = np.tile(np.arange(c.H, dtype=np.uint16), (c.E, 1))
    assert sim.b2m_set_input_perm(c.h, 0, perm.ctypes.data) == L.B2M_EUNSUPPORTED
    assert "llama4" in c.err(), c.err()
    lg = np.zeros((T, c.E), dtype=np.float32)          # logits (kind 1) are fine
    assert sim.b2m_route(c.h, 0, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == 0, c.err()
    c.close()


@needs_sim
def test_expert_parallel_is_refused_on_cpu(sim):
    c = _llama4(sim, max_tokens=64)
    assert c.rc == 0, c.err()
    send = np.zeros((2, 8, c.H), dtype=np.uint16)
    cnt = np.zeros(c.E, dtype=np.int32)
    assert sim.b2m_ep_pack(c.h, 2, 0, 8, 4, send.ctypes.data, cnt.ctypes.data, None) == L.B2M_EUNSUPPORTED
    assert "llama4" in c.err(), c.err()
    handle = (C.c_uint8 * 64)()
    assert sim.b2m_ep_p2p_init(c.h, 2, 0, 8, handle) == L.B2M_EUNSUPPORTED
    c.close()


@needs_sim
@pytest.mark.parametrize("numerics,mode", [(L.NUMERICS_REFERENCE, 6), (L.NUMERICS_FP32, 3)])
def test_combine_mode_and_launch_count_on_cpu(sim, numerics, mode):
    lg = np.random.default_rng(1).standard_normal((5, 8)).astype(np.float32)
    c = _llama4(sim, num_slots=3 * 8, numerics=numerics)
    assert c.rc == 0, c.err()
    c.register_all()
    for l in range(c.L):
        _register_shared(c, l)
    c.forward(0, lg)                                     # the first forward of a layer also uploads its slot table
    take_log(sim)
    s0 = c.stats()["kernel_launches"]
    assert c.forward(0, lg) == 0, c.err()
    log = take_log(sim)
    # COMBINE_LLAMA4 (6), or COMBINE_FP32 (3) for the fp32 numerics; no shared-gate phase (mode 5)
    assert [ln for ln in log if ln.startswith("combine")] == [f"combine T=5 mode={mode} shared=1 ep_collect=0 dtype=0"], log
    n_llama4 = c.stats()["kernel_launches"] - s0
    c.close()
    # the same forward of an ungated DeepSeek shared-expert layer launches as many kernels
    d = Ctx(sim, router=L.ROUTER_DEEPSEEK_GREEDY, expert_type=L.EXPERT_DEEPSEEK, shared_inter=128, num_slots=3 * 8,
            numerics=numerics)
    assert d.rc == 0, d.err()
    d.register_all()
    _register_shared(d, 0)
    d.forward(0, lg)
    take_log(sim)
    s0 = d.stats()["kernel_launches"]
    assert d.forward(0, lg) == 0, d.err()
    take_log(sim)
    assert n_llama4 == d.stats()["kernel_launches"] - s0
    d.close()


# ---------------------------------------------------------------- hf.patch_llama4 on a tiny CPU model
class _RecordingEngine:
    """Records what patch_llama4 hands an engine (the real one needs a GPU)."""

    def __init__(self, I):
        self.router, self.expert_type, self.shared_inter = L.ROUTER_LLAMA4, L.EXPERT_DEEPSEEK, I
        self.fp8 = self.int4 = False
        self.experts, self.registered, self.shared = {}, {}, {}

    def load_expert(self, l, e, ws, **kw):
        self.experts[(l, e)] = [w.clone() for w in ws]

    def register_expert(self, l, e, ws, **kw):
        self.registered[(l, e)] = [w.clone() for w in ws]

    def register_shared(self, l, ws):
        self.shared[l] = [w.clone() for w in ws]


def _tiny_llama4():
    tr = pytest.importorskip("transformers")
    cfg = tr.Llama4TextConfig(vocab_size=128, hidden_size=64, intermediate_size=32, intermediate_size_mlp=96,
                              num_hidden_layers=4, num_attention_heads=2, num_key_value_heads=1, head_dim=32,
                              num_local_experts=4, num_experts_per_tok=1, interleave_moe_layer_step=2,
                              max_position_embeddings=64)
    torch.manual_seed(0)
    model = tr.Llama4ForCausalLM(cfg).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(torch.randn_like(p))
    return model


@pytest.mark.parametrize("resident", [True, False])
def test_patch_llama4_splits_and_transposes(resident):
    model = _tiny_llama4()
    I = model.config.intermediate_size
    layers = model.model.layers
    moe = {l: layers[l].feed_forward for l in range(4)}
    eng = _RecordingEngine(I)
    assert hf.patch_llama4(model, resident=resident, engine=eng) is eng
    kinds = [type(layer.feed_forward).__name__ for layer in layers]
    assert kinds == ["Llama4TextMLP", "B200Llama4MoeAdapter", "Llama4TextMLP", "B200Llama4MoeAdapter"]
    got = eng.experts if resident else eng.registered
    assert sorted(got) == [(l, e) for l in (1, 3) for e in range(4)]
    for l in (1, 3):
        gu, dn = moe[l].experts.gate_up_proj.data, moe[l].experts.down_proj.data
        for e in range(4):
            g, u, d = got[(l, e)]
            assert g.shape == (I, 64) and u.shape == (I, 64) and d.shape == (64, I)
            assert torch.equal(g, gu[e][:, :I].T) and torch.equal(u, gu[e][:, I:].T) and torch.equal(d, dn[e].T)
            assert g.is_contiguous() and u.is_contiguous() and d.is_contiguous()
        sh = moe[l].shared_expert
        assert all(torch.equal(a, b.weight) for a, b in zip(eng.shared[l], (sh.gate_proj, sh.up_proj, sh.down_proj)))
        assert torch.equal(layers[l].feed_forward.gate_weight, moe[l].router.weight)
    assert sorted(eng.shared) == [1, 3]


def test_patch_llama4_refuses_other_engines():
    model = _tiny_llama4()
    eng = _RecordingEngine(model.config.intermediate_size)
    eng.router = L.ROUTER_QWEN_MOE
    with pytest.raises(ValueError, match="ROUTER_LLAMA4"):
        hf.patch_llama4(model, engine=eng)
    eng = _RecordingEngine(model.config.intermediate_size * 2)
    with pytest.raises(ValueError, match="shared_inter"):
        hf.patch_llama4(model, engine=eng)
