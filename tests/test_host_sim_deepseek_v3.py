"""CPU: the C-ABI layer's handling of the DeepSeek-V3 router (B2M_ROUTER_DEEPSEEK_V3) on the host simulation of
tests/test_host_sim.py (api.cu compiled unchanged against stand-in launchers): which configurations b2m_ctx_create_ex
accepts, the argument checks of b2m_set_gate_bias, the missing-bias state error of every routing kind, and the look-ahead
prediction that waits for the next layer's bias."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from moe_infinity_b200 import _lib as L
from test_host_sim import Ctx, _SO, sim  # noqa: F401  (sim: the module-scoped library fixture)

pytestmark = pytest.mark.skipif(_SO is None, reason="nvcc / g++ not available to build the host simulation")


def _v3(lib, **kw):
    kw.setdefault("E", 8)
    kw.setdefault("n_group", 4)
    kw.setdefault("topk_group", 2)
    return Ctx(lib, router=L.ROUTER_DEEPSEEK_V3, expert_type=L.EXPERT_DEEPSEEK, norm_topk_prob=1,
               gate_dtype=L.DTYPE_F32, **kw)


def _bias(E, v=-0.05):
    return np.full(E, v, dtype=np.float32)


def test_v3_router_is_accepted_on_cpu(sim):
    for E, k, n_group, topk_group in ((8, 2, 4, 2), (256, 8, 8, 4), (64, 8, 1, 1), (64, 4, 32, 32), (16, 4, 8, 8)):
        c = _v3(sim, E=E, k=k, n_group=n_group, topk_group=topk_group)
        assert c.rc == 0, (E, k, n_group, topk_group, c.err())
        c.close()


@pytest.mark.parametrize("E,n_group,topk_group,what", [
    (8, 0, 1, "n_group"), (64, 33, 1, "n_group"), (8, 3, 1, "divide"), (8, 8, 1, "at least 2 experts"),
    (256, 256, 1, "n_group"), (8, 4, 0, "topk_group"), (8, 4, 5, "topk_group")])
def test_v3_router_refuses_bad_groups_on_cpu(sim, E, n_group, topk_group, what):
    c = _v3(sim, E=E, n_group=n_group, topk_group=topk_group)
    assert c.rc == L.B2M_EINVAL
    msg = (sim.b2m_last_error(None) or b"").decode()
    assert "deepseek_v3" in msg and what in msg, msg


def test_set_gate_bias_arguments_on_cpu(sim):
    c = _v3(sim)
    assert c.rc == 0, c.err()
    b = _bias(c.E)
    assert sim.b2m_set_gate_bias(c.h, -1, b.ctypes.data) == L.B2M_EINVAL
    assert sim.b2m_set_gate_bias(c.h, c.L, b.ctypes.data) == L.B2M_EINVAL and "out of range" in c.err()
    assert sim.b2m_set_gate_bias(c.h, 0, None) == L.B2M_EINVAL and "null" in c.err()
    assert sim.b2m_set_gate_bias(c.h, 0, b.ctypes.data) == 0, c.err()
    c.close()
    for router in (L.ROUTER_MIXTRAL, L.ROUTER_DEEPSEEK_GREEDY, L.ROUTER_DEEPSEEK_GROUP):
        m = Ctx(sim, router=router, n_group=4, topk_group=2)
        assert m.rc == 0, m.err()
        assert sim.b2m_set_gate_bias(m.h, 0, b.ctypes.data) == L.B2M_EINVAL
        assert "deepseek_v3" in m.err(), m.err()
        m.close()


def test_route_without_bias_is_a_state_error_on_cpu(sim):
    c = _v3(sim, num_slots=3 * 8)
    assert c.rc == 0, c.err()
    T = 5
    x = np.zeros((T, c.H), dtype=np.uint16)
    gate = np.zeros((c.E, c.H), dtype=np.float32)
    lg = np.random.default_rng(0).standard_normal((T, c.E)).astype(np.float32)
    sc = (1 / (1 + np.exp(-lg))).astype(np.float32)
    assert sim.b2m_set_gate(c.h, 0, gate.ctypes.data) == 0
    for kind, rin in ((0, None), (1, lg.ctypes.data), (2, sc.ctypes.data)):
        rc = sim.b2m_route(c.h, 0, x.ctypes.data, rin, kind, L.DTYPE_F32, T, 0, None)
        assert rc == L.B2M_ESTATE, kind
        assert "layer 0 has no correction bias" in c.err(), c.err()
    b = _bias(c.E)
    assert sim.b2m_set_gate_bias(c.h, 0, b.ctypes.data) == 0
    for kind, rin in ((0, None), (1, lg.ctypes.data), (2, sc.ctypes.data)):
        assert sim.b2m_route(c.h, 0, x.ctypes.data, rin, kind, L.DTYPE_F32, T, 0, None) == 0, c.err()
    # the bias is per layer: layer 1 still has none
    assert sim.b2m_route(c.h, 1, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == L.B2M_ESTATE
    c.close()


def test_lookahead_waits_for_next_layers_bias_on_cpu(sim):
    """Offload mode with lookahead_prefetch: the prediction for layer l+1 needs l+1's gate AND bias; without the bias the
    routing call still succeeds and simply makes no prediction."""
    Ln, E = 3, 8
    c = _v3(sim, L_=Ln, E=E, num_slots=10, lookahead_prefetch=2)
    assert c.rc == 0, c.err()
    c.register_all(1)
    gates = [np.random.default_rng(l).standard_normal((E, c.H)).astype(np.float32) for l in range(Ln)]
    biases = [_bias(E, -0.01 * (l + 1)) for l in range(Ln)]
    for l in range(Ln):
        assert sim.b2m_set_gate(c.h, l, gates[l].ctypes.data) == 0
    assert sim.b2m_set_gate_bias(c.h, 0, biases[0].ctypes.data) == 0
    lg = np.random.default_rng(7).standard_normal((4, E)).astype(np.float32)
    look = (C.c_int32 * E)()
    assert c.forward(0, lg) == 0, c.err()
    assert sim.b2m_last_lookahead(c.h, look) == L.B2M_ESTATE          # layer 1 has no bias yet: no prediction
    assert sim.b2m_set_gate_bias(c.h, 1, biases[1].ctypes.data) == 0
    assert c.forward(0, lg) == 0, c.err()
    assert sim.b2m_last_lookahead(c.h, look) == 0, c.err()
    assert sum(look) == 4 * c.k
    c.close()
