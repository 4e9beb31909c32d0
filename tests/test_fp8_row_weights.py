"""CPU: fp8 expert weights with one fp32 scale per output channel (B2M_WEIGHTS_FP8_E4M3_ROW,
moe-infinity_b200/csrc/fp8_weights.cuh and moe_infinity_b200/fp8.py).

* the header's per-row decode equals torch's (q.float() * s[:, None]).to(torch.bfloat16) bit for bit for all 256 e4m3
  codes, under scales whose products are normal, bf16-subnormal, overflow to Inf, and NaN codes; blob sizes;
* quantize_row / dequantize_row: exact round trip on the e4m3 grid, all-zero rows, shape and dtype checks;
* b2m_ctx_create_ex(..., 7, ...) through the host simulation of the C-ABI layer (tests/host/sim): accepted and refused
  configurations with their messages, slot size 3HI + 4(2I + H) rounded up to 16, blob size checks, expert parallelism
  refused, row-format-sized staging copies, and the routed arena's tensor maps against hand-written values;
* the built library has one row-format GEMM per tile width, with the e4m3 -> f16 conversion and register-A HGMMAs."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from moe_infinity_b200.fp8 import dequantize_row, expert_blob_bytes, quantize_row  # noqa: E402

FP8 = torch.float8_e4m3fn
ROW = L.WEIGHTS_FP8_E4M3_ROW


def _f32_bits(x: float) -> str:
    return "%08x" % int(np.array([x], dtype=np.float32).view(np.uint32)[0])


# per-row scales: ordinary ones, products that are bf16 subnormals, fp32 subnormal scales, products that overflow to Inf,
# a negative and a zero scale, and a NaN scale (every product NaN)
SCALES = [1.0, 0.5, 0.0123, 1 / 448, 3.7e5, 2.0 ** -30, 2.0 ** 10, 2.0 ** -120, 1.5 * 2.0 ** -127, 3e-42, 7.5e35, 3.0e37,
          -0.75, 0.0, float("nan")]


def _bf16_bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16).to(torch.int32) & 0xffff


def _is_nan(bits: torch.Tensor) -> torch.Tensor:
    return (((bits >> 7) & 0xff) == 0xff) & ((bits & 0x7f) != 0)


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_host_row_decode_matches_torch(tmp_path):
    exe = tmp_path / "fp8_row_weights_check"
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "moe-infinity_b200", "csrc"),
                    os.path.join(HERE, "host", "fp8_row_weights_check.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)] + [_f32_bits(s) for s in SCALES], capture_output=True, text=True, timeout=60, check=True)
    lines = r.stdout.strip().split("\n")
    got = torch.tensor([[int(v, 16) for v in ln.split()[1:]] for ln in lines[:len(SCALES)]], dtype=torch.int32)
    q = torch.arange(256, dtype=torch.uint8).view(FP8).expand(len(SCALES), 256).contiguous()
    s = torch.tensor(SCALES, dtype=torch.float32)
    want = _bf16_bits((q.float() * s[:, None]).to(torch.bfloat16))
    assert torch.equal(_bf16_bits(dequantize_row(q, s)), want)                 # fp8.py is the same contract
    nan = _is_nan(want)
    assert torch.equal(got[~nan], want[~nan]), (got != want).nonzero()[:8].tolist()
    assert bool(_is_nan(got[nan]).all()), "NaN codes and NaN scales must give NaN"
    # the table reaches both ends of bf16 and NaN: subnormal results, Inf, NaN codes, and a NaN row
    assert bool(((want & 0x7fff) > 0).logical_and((want & 0x7fff) < 0x80).any())
    assert bool(((want & 0x7fff) == 0x7f80).any())
    assert bool(_is_nan(got[-1]).all()) and int(nan[0].sum()) == 2
    tail = dict(ln.split(" ", 1) for ln in lines[len(SCALES):])
    assert tail["blob"].split() == [str(expert_blob_bytes(4096, 14336, "row")), str(expert_blob_bytes(5120, 8192, "row")),
                                    str(expert_blob_bytes(2048, 1408, "row"))]
    assert tail["blob"].split()[0] == str(3 * 4096 * 14336 + 4 * (2 * 14336 + 4096))
    assert tail["vector"] == str(14336 * 4)


def test_quantize_row_roundtrip_and_checks():
    g = torch.Generator().manual_seed(0)
    rows, cols = 256, 384
    codes = torch.randint(0, 256, (rows, cols), generator=g, dtype=torch.uint8)
    codes[(codes & 0x7f) == 0x7f] = 0x38                          # no NaN codes
    codes[:, 5] = 0x7e                                            # every row holds +448: amax / 448 = the row's scale
    s = torch.exp2(torch.randint(-12, 8, (rows,), generator=g).float())
    w = dequantize_row(codes.view(FP8), s, torch.float32)
    q2, s2 = quantize_row(w)
    assert s2.shape == (rows,) and s2.dtype == torch.float32 and torch.equal(s2, s)
    assert torch.equal(q2.view(torch.uint8)[(codes & 0x7f) != 0], codes[(codes & 0x7f) != 0])
    assert torch.equal(dequantize_row(q2, s2.reshape(rows, 1), torch.float32), w)    # [out, 1] scales too
    z = torch.zeros(3, 128)
    z[1] = torch.linspace(-3, 3, 128)
    qz, sz = quantize_row(z)
    assert sz[0].item() == 1.0 and sz[2].item() == 1.0            # an all-zero row gets s = 1 (and zero codes)
    assert torch.equal(qz[0].float(), torch.zeros(128)) and qz[1].float().abs().max().item() == 448.0
    with pytest.raises(ValueError):
        quantize_row(torch.zeros(128))
    with pytest.raises(ValueError):
        dequantize_row(qz, sz[:2])
    with pytest.raises(ValueError):
        dequantize_row(qz, sz.double())
    with pytest.raises(ValueError):
        dequantize_row(qz.float(), sz)
    with pytest.raises(ValueError):
        expert_blob_bytes(256, 512, "col")


# ---------------------------------------------------------------- C-ABI layer through the host simulation
_SO = build_sim.build()
_OBJS = [os.path.join(build_sim.OUT, n) for n in ("api.o", "fake_kernels.o", "fake_cudart.o", "store_reader.o")]


@pytest.fixture(scope="module")
def sim():
    if _SO is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    lib = C.CDLL(_SO)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.b2m_sim_h2d_bytes.restype = C.c_longlong
    lib.b2m_sim_set_total_mem.argtypes = [C.c_longlong]
    return lib


def _cfg(**kw):
    cfg = L.Config()
    cfg.struct_size = C.sizeof(L.Config)
    cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = 2, 8, 256, 512, 2
    cfg.dtype, cfg.expert_type, cfg.router, cfg.max_tokens = L.DTYPE_BF16, L.EXPERT_MIXTRAL, L.ROUTER_MIXTRAL, 64
    cfg.gate_dtype = L.DTYPE_BF16
    cfg.routed_scaling_factor = 1.0
    cfg.num_slots = 16
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _create(lib, fmt=ROW, **kw):
    h = C.c_void_p()
    rc = lib.b2m_ctx_create_ex(C.byref(_cfg(**kw)), fmt, C.byref(h))
    return rc, h


def _stats(lib, h):
    s = L.Stats()
    assert lib.b2m_stats_get(h, C.byref(s)) == 0
    return s.as_dict()


def test_create_ex_accepts_and_refuses(sim):
    llama4 = dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_LLAMA4, top_k=1, shared_inter=512,
                  n_group=1, topk_group=1)
    for kw in (dict(), dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, gate_dtype=L.DTYPE_F32),
               dict(hidden=4096, inter=14336, num_slots=2), dict(hidden=2048, inter=1408, num_slots=2, gemm_impl=2), llama4):
        rc, h = _create(sim, **kw)
        assert rc == 0, (kw, sim.b2m_last_error(None))
        sim.b2m_ctx_destroy(h)
    refused = [(dict(dtype=L.DTYPE_F16, gate_dtype=L.DTYPE_F16), b"bf16"),
               (dict(dtype=L.DTYPE_F32), b"bf16"),
               (dict(hidden=4104), b"multiples of 128"),
               (dict(inter=520), b"multiples of 128"),
               (dict(gemm_impl=1), b"gemm_impl")]
    refused += [(dict(expert_type=t), b"expert_type") for t in range(4)]
    for kw, msg in refused:
        rc, _ = _create(sim, **kw)
        err = sim.b2m_last_error(None)
        assert rc == L.B2M_EUNSUPPORTED, kw
        assert msg in err and b"fp8 (row scales)" in err, (kw, err)
    for fmt in (2, 3, 5, 8):
        assert _create(sim, fmt=fmt)[0] == L.B2M_EINVAL
    assert _create(sim, dtype=L.DTYPE_FP8)[0] == L.B2M_EUNSUPPORTED


@pytest.mark.parametrize("H,I", [(256, 512), (384, 1024), (4096, 14336)])
def test_slot_size_and_blob_checks(sim, H, I):
    blob = expert_blob_bytes(H, I, "row")
    assert blob == (3 * H * I + 4 * (2 * I + H) + 15) // 16 * 16
    rc, h = _create(sim, hidden=H, inter=I, num_slots=2)
    assert rc == 0, sim.b2m_last_error(None)
    try:
        assert _stats(sim, h)["slot_bytes"] == blob
        small = np.zeros(expert_blob_bytes(H, I), dtype=np.uint8)          # the block format's blob
        assert sim.b2m_register_expert(h, 0, 0, small.ctypes.data, small.nbytes) == L.B2M_EINVAL
        ok = np.zeros(blob, dtype=np.uint8)
        assert sim.b2m_register_expert(h, 0, 0, ok.ctypes.data, ok.nbytes) == 0
        # expert parallelism is refused on a row-format context
        assert sim.b2m_ep_pack(h, 2, 0, 64, 8, None, None, None) == L.B2M_EUNSUPPORTED
        hd = (C.c_uint8 * 64)()
        assert sim.b2m_ep_p2p_init(h, 2, 0, 16, hd) == L.B2M_EUNSUPPORTED
        assert b"fp8 (row scales)" in sim.b2m_last_error(h)
    finally:
        sim.b2m_ctx_destroy(h)


def test_offload_stages_row_sized_copies(sim):
    H, I, E = 256, 512, 8
    blob = expert_blob_bytes(H, I, "row")
    rc, h = _create(sim, num_slots=3)
    assert rc == 0
    rng = np.random.default_rng(0)
    blobs = [[rng.integers(0, 255, blob, dtype=np.uint8) for _ in range(E)] for _ in range(2)]
    for l in range(2):
        for e in range(E):
            assert sim.b2m_register_expert(h, l, e, blobs[l][e].ctypes.data, blob) == 0
    h2d0 = sim.b2m_sim_h2d_bytes()
    x = np.zeros((8, H), dtype=np.uint16)
    out = np.zeros_like(x)
    for l in range(2):
        lg = rng.standard_normal((8, E)).astype(np.float32)
        assert sim.b2m_moe_forward(h, l, x.ctypes.data, lg.ctypes.data, 1, L.DTYPE_F32, 8, 0, out.ctypes.data, None) == 0
    st = _stats(sim, h)
    assert st["misses"] > 3 and st["evictions"] > 0
    assert st["h2d_bytes"] == st["misses"] * blob
    staged = sim.b2m_sim_h2d_bytes() - h2d0
    assert staged >= st["misses"] * blob and staged < st["misses"] * blob + 4096   # (+ slot-table and count uploads)
    for e in range(E):
        if sim.b2m_is_resident(h, 1, e) == 1:
            p = C.c_void_p()
            assert sim.b2m_expert_dev_ptr(h, 1, e, C.byref(p)) == 0
            assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * blob).from_address(p.value)), blobs[1][e])
    sim.b2m_ctx_destroy(h)


# ---------------------------------------------------------------- tensor maps (tests/host/sim/tensor_map_probe.cpp)
@pytest.fixture(scope="module")
def map_sim(tmp_path_factory):
    """The host simulation's objects relinked with the tensor-map probe (-Wl,--wrap=cudaGetDriverEntryPoint)."""
    global _SO
    if _SO is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    if not all(os.path.exists(o) for o in _OBJS):     # objects of an older build removed: build the simulation afresh
        os.remove(_SO)
        _SO = build_sim.build()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(build_sim._nvcc())), "include")
    inc = ["-I", build_sim.CSRC, "-I", os.path.join(build_sim.ROOT, "include"), "-I", cuda_inc]
    out = tmp_path_factory.mktemp("row_map_probe")
    obj, so = str(out / "tensor_map_probe.o"), str(out / "libb2m_hostsim_row_map_probe.so")
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


UINT8, SW64 = 0, 2   # CUtensorMapDataType / CUtensorMapSwizzle values (cuda.h)


@pytest.mark.parametrize("model", ["mixtral", "deepseek"])
def test_routed_arena_maps(map_sim, model):
    H, I, SLOTS = 256, 512, 4
    slot = 3 * H * I + 4 * (2 * I + H)                  # 398336, a multiple of 16
    # Mixtral stores w1 | w2 | w3 (gate, down, up), DeepSeek gate | up | down; the scale vectors follow and are not mapped
    off_gate, off_up, off_down = (0, 262144, 131072) if model == "mixtral" else (0, 131072, 262144)
    kw = (dict(expert_type=L.EXPERT_MIXTRAL, router=L.ROUTER_MIXTRAL, gate_dtype=L.DTYPE_BF16) if model == "mixtral" else
          dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, gate_dtype=L.DTYPE_F32))
    _take_maps(map_sim)
    h = C.c_void_p()
    assert map_sim.b2m_ctx_create_ex(C.byref(_cfg(num_slots=SLOTS, **kw)), ROW, C.byref(h)) == 0, map_sim.b2m_last_error(None)
    try:
        maps = [m for m in _take_maps(map_sim) if len(m["dims"]) == 3]
        assert len(maps) == 6, maps       # gate, up, down with 128-row boxes, then with 64-row boxes
        arena = maps[0]["base"]
        for i, m in enumerate(maps):
            which = i % 3
            assert m["dt"] == UINT8 and m["swz"] == SW64, (i, m)
            assert m["box"] == (64, 128 if i < 3 else 64, 1), (i, m)
            if which < 2:   # gate / up: [I rows][H k], one byte each
                assert m["dims"] == (H, I, SLOTS) and m["strides"] == (H, slot), (i, m)
                assert m["base"] - arena == (off_gate, off_up)[which], (i, m)
            else:           # down: [H rows][I k]
                assert m["dims"] == (I, H, SLOTS) and m["strides"] == (I, slot), (i, m)
                assert m["base"] - arena == off_down, (i, m)
        assert _stats(map_sim, h)["slot_bytes"] == slot
    finally:
        map_sim.b2m_ctx_destroy(h)


def test_library_has_fp8_row_sass(lib_built):
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    fns = sass.split("Function : ")
    row = [f for f in fns if f.startswith("_ZN3b2m27grouped_gemm_fp8_row_kernel")]
    assert len(row) == 9, "one row-format instantiation per tile width (gate/up 16..128, down 16..256)"
    for f in row:
        assert "F2FP.F16.E4M3" in f
        # register-A wgmma: HGMMA's A operand is a register, B a shared-memory descriptor
        assert any(ln.split("HGMMA", 1)[1].split(",")[1].strip().startswith("R") for ln in f.split("\n") if "HGMMA" in ln)
