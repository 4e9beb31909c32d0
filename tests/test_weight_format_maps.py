"""CPU: the TMA maps of the routed experts' slot arena for every weight format, through the host simulation.

The GEMM kernels read each expert matrix through a 3-D tensor map {k, rows, slot}: for each format the map's element type,
swizzle, extents, strides and box must agree with the format's tile layout (fp8_weights.cuh, int4_weights.cuh), and its base
with the slot layout.  A CPU cannot run TMA, so a copy of the host simulation linked with tests/host/sim/tensor_map_probe.cpp
records what b2m_ctx_create_ex hands to cuTensorMapEncodeTiled, and this test checks it against values written out by hand
for H = 256, I = 512 and 4 slots."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402

_SO = build_sim.build()
_OBJS = [os.path.join(build_sim.OUT, n) for n in ("api.o", "fake_kernels.o", "fake_cudart.o", "store_reader.o")]
pytestmark = pytest.mark.skipif(_SO is None, reason="nvcc / g++ not available to build the host simulation")

H, I, SLOTS = 256, 512, 4
# CUtensorMapDataType / CUtensorMapSwizzle values (cuda.h)
UINT8, FLOAT16, BFLOAT16 = 0, 6, 9
SW32, SW64, SW128 = 1, 2, 3

# format, model dtype -> (element type, swizzle, slot bytes, row bytes of gate/up, of down, k extent of gate/up, of down,
# box width)
GEOMETRY = {
    "bf16": (L.WEIGHTS_MODEL_DTYPE, L.DTYPE_BF16, BFLOAT16, SW128, 786432, 512, 1024, 256, 512, 64),
    "f16": (L.WEIGHTS_MODEL_DTYPE, L.DTYPE_F16, FLOAT16, SW128, 786432, 512, 1024, 256, 512, 64),
    "fp8": (L.WEIGHTS_FP8_E4M3_B128, L.DTYPE_BF16, UINT8, SW64, 393312, 256, 512, 256, 512, 64),
    "int4": (L.WEIGHTS_INT4_G128, L.DTYPE_BF16, UINT8, SW32, 208896, 128, 256, 128, 256, 32),
    "int4_f16": (L.WEIGHTS_INT4_G128_F16, L.DTYPE_F16, UINT8, SW32, 208896, 128, 256, 128, 256, 32),
}
# byte offsets of gate, up and down in a slot: Mixtral stores w1 | w2 | w3 (gate, down, up), DeepSeek gate | up | down
OFFSETS = {
    ("bf16", "mixtral"): (0, 524288, 262144), ("bf16", "deepseek"): (0, 262144, 524288),
    ("f16", "mixtral"): (0, 524288, 262144), ("f16", "deepseek"): (0, 262144, 524288),
    ("fp8", "mixtral"): (0, 262144, 131072), ("fp8", "deepseek"): (0, 131072, 262144),
    ("int4", "mixtral"): (0, 131072, 65536), ("int4", "deepseek"): (0, 65536, 131072),
    ("int4_f16", "mixtral"): (0, 131072, 65536), ("int4_f16", "deepseek"): (0, 65536, 131072),
}


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    """The host simulation's objects relinked with the tensor-map probe (-Wl,--wrap=cudaGetDriverEntryPoint)."""
    global _SO
    if not all(os.path.exists(o) for o in _OBJS):     # objects of an older build removed: build the simulation afresh
        os.remove(_SO)
        _SO = build_sim.build()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(build_sim._nvcc())), "include")
    inc = ["-I", build_sim.CSRC, "-I", os.path.join(build_sim.ROOT, "include"), "-I", cuda_inc]
    out = tmp_path_factory.mktemp("map_probe")
    obj, so = str(out / "tensor_map_probe.o"), str(out / "libb2m_hostsim_map_probe.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", *inc, "-c", os.path.join(HERE, "host", "sim", "tensor_map_probe.cpp"),
                    "-o", obj], check=True, capture_output=True)
    subprocess.run(["g++", "-shared", "-Wl,-Bsymbolic", "-Wl,--wrap=cudaGetDriverEntryPoint", "-o", so, *_OBJS, obj,
                    "-lpthread"], check=True, capture_output=True)
    lib = C.CDLL(so)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.b2m_probe_take_maps.restype, lib.b2m_probe_take_maps.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t]
    return lib


def _take_maps(lib):
    buf = C.create_string_buffer(1 << 20)
    lib.b2m_probe_take_maps(buf, len(buf))
    maps = []
    for ln in buf.value.decode().split("\n"):
        if ln:
            f = dict(kv.split("=") for kv in ln.split())
            maps.append({k: int(v) if k in ("dt", "swz", "base") else tuple(int(x) for x in v.split(",")) for k, v in f.items()})
    return maps


@pytest.mark.parametrize("model", ["mixtral", "deepseek"])
@pytest.mark.parametrize("fmt", list(GEOMETRY))
def test_routed_arena_maps(sim, fmt, model):
    wf, dtype, dt, swz, slot, row_up, row_dn, k_up, k_dn, box_k = GEOMETRY[fmt]
    cfg = L.Config()
    cfg.struct_size = C.sizeof(L.Config)
    cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = 2, 8, H, I, 2
    cfg.dtype, cfg.max_tokens, cfg.num_slots, cfg.routed_scaling_factor = dtype, 64, SLOTS, 1.0
    if model == "mixtral":
        cfg.expert_type, cfg.router, cfg.gate_dtype = L.EXPERT_MIXTRAL, L.ROUTER_MIXTRAL, dtype
    else:
        cfg.expert_type, cfg.router, cfg.gate_dtype = L.EXPERT_DEEPSEEK, L.ROUTER_DEEPSEEK_GREEDY, L.DTYPE_F32
    _take_maps(sim)
    h = C.c_void_p()
    assert sim.b2m_ctx_create_ex(C.byref(cfg), wf, C.byref(h)) == 0, sim.b2m_last_error(None)
    try:
        maps = [m for m in _take_maps(sim) if len(m["dims"]) == 3]
        # gate, up, down with 128-row boxes, then with 64-row boxes; no other 3-D map without shared experts
        assert len(maps) == 6, maps
        arena = maps[0]["base"]
        off_gate, off_up, off_down = OFFSETS[(fmt, model)]
        for i, m in enumerate(maps):
            rows = 128 if i < 3 else 64
            which = i % 3
            assert m["dt"] == dt and m["swz"] == swz, (i, m)
            assert m["box"] == (box_k, rows, 1), (i, m)
            if which < 2:   # gate / up: [I rows][H k]
                assert m["dims"] == (k_up, I, SLOTS) and m["strides"] == (row_up, slot), (i, m)
                assert m["base"] - arena == (off_gate, off_up)[which], (i, m)
            else:           # down: [H rows][I k]
                assert m["dims"] == (k_dn, H, SLOTS) and m["strides"] == (row_dn, slot), (i, m)
                assert m["base"] - arena == off_down, (i, m)
        s = L.Stats()
        assert sim.b2m_stats_get(h, C.byref(s)) == 0
        assert s.as_dict()["slot_bytes"] == slot
    finally:
        sim.b2m_ctx_destroy(h)
