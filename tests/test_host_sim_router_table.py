"""CPU: what each router kind (B2M_ROUTER_*) admits and changes in the C-ABI layer, for all seven kinds, on the host
simulation of tests/test_host_sim.py (api.cu compiled unchanged against stand-in launchers).  The expected values are
written out literally; they pin the router table in api.cu to the behaviour of the per-router branches it replaced:
  * b2m_ctx_create_ex's return code over a fixed grid of configurations;
  * which of b2m_set_gate_bias, b2m_set_shared_gate, b2m_set_input_perm (on an f16 int4 context), scores as router input
    and the expert-parallel entry points each kind accepts;
  * the combine mode of both numerics, kernel_launches of one forward at T <= 256 and at T > 256, and the routing launch's
    scale_rows and logits_model_dtype (recorded by tests/host/sim/route_flags_probe.cpp in a relinked copy of the
    simulation)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from test_host_sim import Ctx, _SO, _kv, sim, take_log  # noqa: E402,F401  (sim: the module-scoped library fixture)

pytestmark = pytest.mark.skipif(_SO is None, reason="nvcc / g++ not available to build the host simulation")
_OBJS = [os.path.join(build_sim.OUT, n) for n in ("api.o", "fake_kernels.o", "fake_cudart.o", "store_reader.o")]
_WRAPPED = "_ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st"


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    """The host simulation's objects relinked with tests/host/sim/route_flags_probe.cpp (-Wl,--wrap on launch_route), which
    records RouteParams::scale_rows and RouteParams::logits_model_dtype of every routing launch."""
    so = _SO
    if not all(os.path.exists(o) for o in _OBJS):     # objects of an older build removed: build the simulation afresh
        os.remove(so)
        so = build_sim.build()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(build_sim._nvcc())), "include")
    inc = ["-I", build_sim.CSRC, "-I", os.path.join(build_sim.ROOT, "include"), "-I", cuda_inc]
    out = tmp_path_factory.mktemp("route_flags_probe")
    obj, so = str(out / "route_flags_probe.o"), str(out / "libb2m_hostsim_route_flags.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", *inc, "-c", os.path.join(HERE, "host", "sim", "route_flags_probe.cpp"),
                    "-o", obj], check=True, capture_output=True)
    subprocess.run(["g++", "-shared", "-Wl,-Bsymbolic", f"-Wl,--wrap={_WRAPPED}", "-o", so, *_OBJS, obj, "-lpthread"],
                   check=True, capture_output=True)
    lib = C.CDLL(so)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.b2m_sim_take_log.restype, lib.b2m_sim_take_log.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t]
    lib.b2m_probe_take_route_flags.restype = C.c_size_t
    lib.b2m_probe_take_route_flags.argtypes = [C.POINTER(C.c_int32), C.c_size_t]
    return lib


def _take_route_flags(lib):
    """(scale_rows, logits_model_dtype) of each routing launch since the last call."""
    buf = (C.c_int32 * 256)()
    n = min(lib.b2m_probe_take_route_flags(buf, 256), 256)
    return [(buf[i], buf[i + 1]) for i in range(0, n, 2)]

OK, EINVAL, ESTATE, EUNSUP = L.B2M_OK, L.B2M_EINVAL, L.B2M_ESTATE, L.B2M_EUNSUPPORTED
ROUTERS = (L.ROUTER_MIXTRAL, L.ROUTER_DEEPSEEK_GREEDY, L.ROUTER_DEEPSEEK_GROUP, L.ROUTER_SWITCH_TOP1, L.ROUTER_DEEPSEEK_V3,
           L.ROUTER_QWEN_MOE, L.ROUTER_LLAMA4)

# A configuration every kind except Switch (top_k 1) accepts, then one field changed at a time.  Columns: the seven kinds
# in B2M_ROUTER_* order (mixtral, greedy, group, switch, deepseek_v3, qwen_moe, llama4).
BASE = dict(E=8, k=2, expert_type=L.EXPERT_DEEPSEEK, n_group=1, topk_group=1, shared_inter=128)
CREATE_CODES = {
    "base":                 (OK, OK, OK, EINVAL, OK, OK, OK),
    "top_k=1":              (OK, OK, OK, OK, OK, OK, OK),
    "expert_type=mixtral":  (OK, OK, OK, EINVAL, OK, EINVAL, EINVAL),
    "dtype=f16":            (OK, OK, OK, EINVAL, OK, OK, OK),
    "dtype=f32":            (OK, OK, OK, EINVAL, OK, EINVAL, EINVAL),
    "groups=0/0":           (OK, OK, OK, EINVAL, EINVAL, EINVAL, EINVAL),
    "groups=2/1":           (OK, OK, OK, EINVAL, OK, EINVAL, EINVAL),
    "groups=1/2":           (OK, OK, OK, EINVAL, EINVAL, EINVAL, EINVAL),
    "groups=3/1":           (OK, OK, OK, EINVAL, EINVAL, EINVAL, EINVAL),
    "groups=8/1":           (OK, OK, OK, EINVAL, EINVAL, EINVAL, EINVAL),
    "groups=4/4":           (OK, OK, OK, EINVAL, OK, EINVAL, EINVAL),
    "groups=33/1":          (OK, OK, OK, EINVAL, EINVAL, EINVAL, EINVAL),
    "scaling=2.5":          (OK, OK, OK, EINVAL, OK, EINVAL, EINVAL),
    "norm=1":               (OK, OK, OK, EINVAL, OK, OK, EINVAL),
    "shared_inter=0":       (OK, OK, OK, EINVAL, OK, OK, EINVAL),
    "top_k=1,mixtral,f32":  (OK, OK, OK, OK, OK, EINVAL, EINVAL),
}
VARIANTS = {
    "base": {}, "top_k=1": dict(k=1), "expert_type=mixtral": dict(expert_type=L.EXPERT_MIXTRAL),
    "dtype=f16": dict(dtype=L.DTYPE_F16, gate_dtype=L.DTYPE_F16), "dtype=f32": dict(dtype=L.DTYPE_F32, gate_dtype=L.DTYPE_F32),
    "groups=0/0": dict(n_group=0, topk_group=0), "groups=2/1": dict(n_group=2), "groups=1/2": dict(topk_group=2),
    "groups=3/1": dict(n_group=3), "groups=8/1": dict(n_group=8), "groups=4/4": dict(n_group=4, topk_group=4),
    "groups=33/1": dict(n_group=33), "scaling=2.5": dict(routed_scaling_factor=2.5), "norm=1": dict(norm_topk_prob=1),
    "shared_inter=0": dict(shared_inter=0),
    "top_k=1,mixtral,f32": dict(k=1, expert_type=L.EXPERT_MIXTRAL, dtype=L.DTYPE_F32, gate_dtype=L.DTYPE_F32),
}
NAMES = ("mixtral", "greedy", "group", "switch", "deepseek_v3", "qwen_moe", "llama4")


def test_create_codes(sim):
    assert sorted(VARIANTS) == sorted(CREATE_CODES)
    for name, want in CREATE_CODES.items():
        got = []
        for router in ROUTERS:
            c = Ctx(sim, router=router, **{**BASE, **VARIANTS[name]})
            got.append(c.rc)
            if c.rc == EINVAL:          # the message names the kind it refused for
                msg = (sim.b2m_last_error(None) or b"").decode()
                assert NAMES[router] in msg, (name, msg)
            c.close()
        assert tuple(got) == want, (name, got)


def test_unknown_router_kind(sim):
    for router in (-1, 7):
        c = Ctx(sim, router=router, **BASE)
        assert c.rc == EINVAL and "router" in (sim.b2m_last_error(None) or b"").decode()
        c.close()


def _good(router, **kw):
    """A configuration `router` accepts (kw overrides it)."""
    cfg = dict(BASE, k=1 if router == L.ROUTER_SWITCH_TOP1 else 2)
    if router in (L.ROUTER_DEEPSEEK_GROUP, L.ROUTER_DEEPSEEK_V3):
        cfg.update(n_group=2, topk_group=1)
    cfg.update(kw)
    return cfg


def _create_ex(lib, fmt, E, k, expert_type, **kw):
    cfg = L.Config()
    cfg.struct_size = C.sizeof(L.Config)
    cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k, cfg.max_tokens = 3, E, 128, 256, k, 64
    cfg.expert_type, cfg.routed_scaling_factor, cfg.num_slots = expert_type, 1.0, 24
    for key, v in kw.items():
        setattr(cfg, key, v)
    h = C.c_void_p()
    assert lib.b2m_ctx_create_ex(C.byref(cfg), fmt, C.byref(h)) == 0, lib.b2m_last_error(None)
    return h


# per kind: set_gate_bias, set_shared_gate, set_input_perm (f16 int4 context), b2m_route with scores, b2m_ep_ungroup
ACCEPTS = {
    L.ROUTER_MIXTRAL:         (EINVAL, EINVAL, OK, OK, OK),
    L.ROUTER_DEEPSEEK_GREEDY: (EINVAL, EINVAL, OK, OK, OK),
    L.ROUTER_DEEPSEEK_GROUP:  (EINVAL, EINVAL, OK, OK, OK),
    L.ROUTER_SWITCH_TOP1:     (EINVAL, EINVAL, OK, OK, OK),
    L.ROUTER_DEEPSEEK_V3:     (OK, EINVAL, OK, OK, OK),
    L.ROUTER_QWEN_MOE:        (EINVAL, OK, OK, OK, EUNSUP),
    L.ROUTER_LLAMA4:          (EINVAL, EINVAL, EUNSUP, EUNSUP, EUNSUP),
}


@pytest.mark.parametrize("router", ROUTERS)
def test_entry_points_each_kind_accepts(sim, router):
    c = Ctx(sim, router=router, **_good(router))
    assert c.rc == 0, c.err()
    bias = np.zeros(c.E, dtype=np.float32)
    gate = np.zeros(c.H, dtype=np.uint16)
    got = [sim.b2m_set_gate_bias(c.h, 0, bias.ctypes.data)]
    assert got[0] == 0 or "deepseek_v3" in c.err(), c.err()      # a refusal names the kind that has the feature
    got.append(sim.b2m_set_shared_gate(c.h, 0, gate.ctypes.data))
    assert got[1] == 0 or "qwen_moe" in c.err(), c.err()
    T = 4
    x = np.zeros((T, c.H), dtype=np.uint16)
    scores = np.full((T, c.E), 1.0 / c.E, dtype=np.float32)
    if router == L.ROUTER_DEEPSEEK_V3:
        assert sim.b2m_route(c.h, 1, x.ctypes.data, scores.ctypes.data, 2, L.DTYPE_F32, T, 0, None) == ESTATE   # no bias on layer 1
    rc = sim.b2m_route(c.h, 0, x.ctypes.data, scores.ctypes.data, 2, L.DTYPE_F32, T, 0, None)
    ret = np.zeros((2, 9, c.H), dtype=np.uint16)
    rc_ep = sim.b2m_ep_ungroup(c.h, 2, 0, 8, ret.ctypes.data, None)
    c.close()
    h = _create_ex(sim, L.WEIGHTS_INT4_G128_F16, router=router, **_good(router, dtype=L.DTYPE_F16, gate_dtype=L.DTYPE_F16))
    perm = np.tile(np.arange(128, dtype=np.uint16), (8, 1))
    got += [sim.b2m_set_input_perm(h, 0, perm.ctypes.data), rc, rc_ep]
    sim.b2m_ctx_destroy(h)
    assert tuple(got) == ACCEPTS[router], got


# per kind: the logged combine modes of one forward under B2M_NUMERICS_REFERENCE and B2M_NUMERICS_FP32 (Qwen's gate phase,
# mode 5, first), the routing launch's scale_rows and logits_model_dtype, kernel_launches of one forward at T = 5 and at
# T = 300, and b2m_moe_forward's code for scores as router input
FORWARD = {
    L.ROUTER_MIXTRAL:         ((0,), (3,), 0, 1, 9, 8, OK),
    L.ROUTER_DEEPSEEK_GREEDY: ((1,), (3,), 0, 0, 9, 8, OK),
    L.ROUTER_DEEPSEEK_GROUP:  ((1,), (3,), 0, 0, 9, 8, OK),
    L.ROUTER_SWITCH_TOP1:     ((2,), (2,), 0, 0, 9, 10, OK),
    L.ROUTER_DEEPSEEK_V3:     ((1,), (3,), 0, 0, 9, 8, OK),
    L.ROUTER_QWEN_MOE:        ((5, 4), (5, 3), 0, 1, 10, 9, OK),
    L.ROUTER_LLAMA4:          ((6,), (3,), 1, 1, 9, 8, EUNSUP),
}


def _forward_ctx(lib, router, numerics):
    c = Ctx(lib, router=router, **_good(router, num_slots=24, max_tokens=512, numerics=numerics))
    assert c.rc == 0, c.err()
    c.register_all()
    blob = np.zeros(3 * c.H * 128 * 2, dtype=np.uint8)
    c.blobs["shared"] = blob
    assert lib.b2m_register_shared(c.h, 0, blob.ctypes.data, blob.nbytes) == 0, c.err()
    c.bias, c.gate = np.zeros(c.E, dtype=np.float32), np.zeros(c.H, dtype=np.uint16)
    if router == L.ROUTER_DEEPSEEK_V3:
        assert lib.b2m_set_gate_bias(c.h, 0, c.bias.ctypes.data) == 0, c.err()
    if router == L.ROUTER_QWEN_MOE:
        assert lib.b2m_set_shared_gate(c.h, 0, c.gate.ctypes.data) == 0, c.err()
    return c


def _launches(c, T):
    lg = np.random.default_rng(T).standard_normal((T, c.E)).astype(np.float32)
    s0 = c.stats()["kernel_launches"]
    assert c.forward(0, lg) == 0, c.err()
    return c.stats()["kernel_launches"] - s0


@pytest.mark.parametrize("router", ROUTERS)
def test_forward_of_each_kind(probe, router):
    sim = probe
    modes_ref, modes_fp32, scale_rows, logits_model_dtype, n_small, n_large, scores_rc = FORWARD[router]
    for numerics, want_modes in ((L.NUMERICS_REFERENCE, modes_ref), (L.NUMERICS_FP32, modes_fp32)):
        c = _forward_ctx(sim, router, numerics)
        _launches(c, 5)                                   # the first forward of a layer also uploads its slot table
        take_log(sim)
        _take_route_flags(sim)
        assert _launches(c, 5) == n_small
        log = take_log(sim)
        assert _take_route_flags(sim) == [(scale_rows, logits_model_dtype)]
        assert tuple(int(_kv(ln)["mode"]) for ln in log if ln.startswith("combine")) == want_modes, log
        route = _kv([ln for ln in log if ln.startswith("route")][0])
        # the gate/up GEMM starts under the permute kernel, except behind Switch's capacity pass
        assert int(route["offsets_early"]) == (0 if router == L.ROUTER_SWITCH_TOP1 else 1), route
        assert _launches(c, 300) == n_large
        T = 4
        x, out = np.zeros((T, c.H), dtype=np.uint16), np.zeros((T, c.H), dtype=np.uint16)
        scores = np.full((T, c.E), 1.0 / c.E, dtype=np.float32)
        assert sim.b2m_moe_forward(c.h, 0, x.ctypes.data, scores.ctypes.data, 2, L.DTYPE_F32, T, 0, out.ctypes.data,
                                   None) == scores_rc, c.err()
        c.close()
