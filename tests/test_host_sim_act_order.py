"""CPU: b2m_set_input_perm through the host simulation (tests/host/sim): accepted on a B2M_WEIGHTS_INT4_G128_F16 context
only, B2M_EINVAL for a layer out of range, and the table reaches RouteParams for the layers that set one, on both routing
entry points, until it is cleared with NULL.  The last check runs on a copy of the simulation linked with
tests/host/sim/route_perm_probe.cpp, which records RouteParams::input_perm of every routing launch api.cu makes."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402

_SO = build_sim.build()
_OBJS = [os.path.join(build_sim.OUT, n) for n in ("api.o", "fake_kernels.o", "fake_cudart.o", "store_reader.o")]
_WRAPPED = ("_ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st",
            "_ZN3b2m22launch_route_from_maskERKNS_11RouteParamsEPKhP11CUstream_st")


def _bind(path):
    lib = C.CDLL(path)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def sim():
    if _SO is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    return _bind(_SO)


@pytest.fixture(scope="module")
def probe():
    """The host simulation's objects relinked with the routing-launch probe (-Wl,--wrap on both routing launchers)."""
    global _SO
    if _SO is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    if not all(os.path.exists(o) for o in _OBJS):     # objects of an older build removed: build the simulation afresh
        os.remove(_SO)
        _SO = build_sim.build()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(build_sim._nvcc())), "include")
    inc = ["-I", build_sim.CSRC, "-I", os.path.join(build_sim.ROOT, "include"), "-I", cuda_inc]
    obj = os.path.join(build_sim.OUT, "route_perm_probe.o")
    so = os.path.join(build_sim.OUT, "libb2m_hostsim_perm_probe.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", *inc, "-c", os.path.join(HERE, "host", "sim", "route_perm_probe.cpp"),
                    "-o", obj], check=True, capture_output=True)
    wrap = [f"-Wl,--wrap={s}" for s in _WRAPPED]
    subprocess.run(["g++", "-shared", "-Wl,-Bsymbolic", *wrap, "-o", so, *_OBJS, obj, "-lpthread"], check=True,
                   capture_output=True)
    lib = _bind(so)
    lib.b2m_probe_take_perms.restype = C.c_size_t
    lib.b2m_probe_take_perms.argtypes = [C.POINTER(C.c_uint64), C.c_size_t]
    return lib


def _create(lib, fmt, dtype):
    cfg = L.Config()
    cfg.struct_size = C.sizeof(L.Config)
    cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = 2, 8, 256, 512, 2
    cfg.dtype, cfg.expert_type, cfg.router, cfg.max_tokens = dtype, L.EXPERT_MIXTRAL, L.ROUTER_MIXTRAL, 64
    cfg.gate_dtype, cfg.routed_scaling_factor, cfg.num_slots = dtype, 1.0, 16
    h = C.c_void_p()
    assert lib.b2m_ctx_create_ex(C.byref(cfg), fmt, C.byref(h)) == 0, lib.b2m_last_error(None)
    return h


def _take_perms(lib):
    buf = (C.c_uint64 * 64)()
    n = lib.b2m_probe_take_perms(buf, 64)
    return list(buf[:min(n, 64)])


def test_set_input_perm_formats_and_layers(sim):
    table = np.tile(np.arange(256, dtype=np.uint16), (8, 1))
    h = _create(sim, L.WEIGHTS_INT4_G128_F16, L.DTYPE_F16)
    assert sim.b2m_set_input_perm(h, 0, table.ctypes.data) == 0
    assert sim.b2m_set_input_perm(h, 1, None) == 0
    for bad in (-1, 2):
        assert sim.b2m_set_input_perm(h, bad, table.ctypes.data) == L.B2M_EINVAL
    sim.b2m_ctx_destroy(h)
    for fmt, dt in ((L.WEIGHTS_MODEL_DTYPE, L.DTYPE_F16), (L.WEIGHTS_MODEL_DTYPE, L.DTYPE_BF16),
                    (L.WEIGHTS_FP8_E4M3_B128, L.DTYPE_BF16), (L.WEIGHTS_INT4_G128, L.DTYPE_BF16)):
        h = _create(sim, fmt, dt)
        assert sim.b2m_set_input_perm(h, 0, table.ctypes.data) == L.B2M_EUNSUPPORTED, fmt
        assert b"B2M_WEIGHTS_INT4_G128_F16" in sim.b2m_last_error(h)
        sim.b2m_ctx_destroy(h)


def test_table_reaches_routing_of_its_layer_only(probe):
    T, H, E = 8, 256, 8
    h = _create(probe, L.WEIGHTS_INT4_G128_F16, L.DTYPE_F16)
    rng = np.random.default_rng(3)
    table = np.stack([rng.permutation(H) for _ in range(E)]).astype(np.uint16)
    x = np.zeros((T, H), dtype=np.uint16)
    logits = rng.standard_normal((T, E)).astype(np.float32)
    mask = np.zeros((T, E), dtype=np.uint8)
    mask[:, :2] = 1

    def tables(layer):
        """input_perm of the launches of one b2m_route and one b2m_route_from_mask call on `layer`."""
        _take_perms(probe)
        assert probe.b2m_route(h, layer, x.ctypes.data, logits.ctypes.data, 1, L.DTYPE_F32, T, 0, None) == 0
        assert probe.b2m_route_from_mask(h, layer, x.ctypes.data, mask.ctypes.data, T, None) == 0
        return _take_perms(probe)

    assert tables(0) == [0, 0] and tables(1) == [0, 0]
    assert probe.b2m_set_input_perm(h, 0, table.ctypes.data) == 0
    assert tables(0) == [table.ctypes.data] * 2
    assert tables(1) == [0, 0]
    assert probe.b2m_set_input_perm(h, 0, None) == 0
    assert tables(0) == [0, 0]
    probe.b2m_ctx_destroy(h)
