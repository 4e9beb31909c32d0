"""CPU: fp8 expert weights (B2M_WEIGHTS_FP8_E4M3_B128, moe-infinity_b200/csrc/fp8_weights.cuh and moe_infinity_b200/fp8.py).

* the header's host dequantisation equals torch's (w_q.float() * s).to(torch.bfloat16) bit for bit for all 256 e4m3 codes,
  with scales whose products round to bf16 subnormals and ones that overflow to Inf; NaN codes give NaN;
* quantize_block128 / dequantize_block128: exact round trip on the e4m3 grid, zero blocks, clamping, non-square grids;
* b2m_ctx_create_ex through the host simulation of the C-ABI layer (tests/host/sim): accepted and refused configurations,
  slot size and count, blob size checks, expert parallelism refused, fp8-sized staging copies;
* the built library's grouped GEMMs contain the e4m3 -> f16 conversion and register-A HGMMAs."""
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
from moe_infinity_b200.fp8 import dequantize_block128, expert_blob_bytes, quantize_block128  # noqa: E402

FP8 = torch.float8_e4m3fn
TOTAL_MEM = 8 << 30   # the simulation's default device memory


def _f32_bits(x: float) -> str:
    return "%08x" % int(np.array([x], dtype=np.float32).view(np.uint32)[0])


# scales: ordinary ones, products that are bf16 subnormals (2^-130 .. 2^-120 times a code), fp32 subnormal scales, and
# products that overflow bf16 / fp32 to Inf
SCALES = [1.0, 0.5, 0.0123, 1 / 448, 3.7e5, 2.0 ** -30, 2.0 ** 10, 2.0 ** -120, 1.5 * 2.0 ** -127, 3e-42, 7.5e35, 3.0e37,
          -0.75, 0.0]


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_host_dequant_matches_torch(tmp_path):
    exe = tmp_path / "fp8_weights_check"
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "moe-infinity_b200", "csrc"),
                    os.path.join(HERE, "host", "fp8_weights_check.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)] + [_f32_bits(s) for s in SCALES], capture_output=True, text=True, timeout=60, check=True)
    lines = r.stdout.strip().split("\n")
    codes = torch.arange(256, dtype=torch.uint8).view(FP8)
    nan = (torch.arange(256) & 0x7f) == 0x7f
    for s, line in zip(SCALES, lines):
        got = torch.tensor([int(v, 16) for v in line.split()[1:]], dtype=torch.int32)
        want = (codes.float() * torch.tensor(s, dtype=torch.float32)).to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xffff
        assert torch.equal(got[~nan], want[~nan]), f"scale {s}: {(got != want).nonzero().flatten().tolist()[:8]}"
        assert bool((((got[nan] >> 7) & 0xff) == 0xff).all() and ((got[nan] & 0x7f) != 0).all()), "NaN codes must give NaN"
    # the scales above reach both ends of bf16: subnormal results and Inf
    assert any(0 < (int(v, 16) & 0x7fff) < 0x80 for ln in lines for v in ln.split()[1:])
    assert any((int(v, 16) & 0x7fff) == 0x7f80 for ln in lines for v in ln.split()[1:])
    tail = dict(ln.split(" ", 1) for ln in lines[len(SCALES):])
    assert tail["blob"].split() == [str(expert_blob_bytes(4096, 14336)), str(expert_blob_bytes(2048, 1408))]
    assert tail["blob"].split()[0] == "176203776"
    m = 2048 * 1408
    g = (2048 // 128) * (1408 // 128) * 4
    assert tail["grid"].split() == [str(3 * m), str(3 * m + g), str(3 * m + 2 * g)]
    assert tail["tile"] == "ok"


def test_quantize_roundtrip_on_grid():
    g = torch.Generator().manual_seed(0)
    rows, cols = 256, 384                                         # a non-square 2 x 3 grid
    codes = torch.randint(0, 256, (rows, cols), generator=g, dtype=torch.uint8)
    codes[(codes & 0x7f) == 0x7f] = 0x38                          # no NaN codes
    codes[::128, ::128] = 0x7e                                    # every block holds +448: amax / 448 = the block's scale
    q = codes.view(FP8)
    s = torch.exp2(torch.tensor([[-3.0, 0.0, 5.0], [2.0, -10.0, 1.0]]))
    w = dequantize_block128(q, s, torch.float32)
    q2, s2 = quantize_block128(w)
    assert s2.shape == (2, 3) and s2.dtype == torch.float32
    assert torch.equal(s2, s)
    assert torch.equal(q2.view(torch.uint8)[(codes & 0x7f) != 0], codes[(codes & 0x7f) != 0])   # (+-0 keep their value)
    assert torch.equal(dequantize_block128(q2, s2, torch.float32), w)


def test_quantize_zero_blocks_and_clamp():
    w = torch.zeros(128, 256)
    w[:, 128:] = torch.linspace(-3, 3, 128 * 128).reshape(128, 128)
    q, s = quantize_block128(w)
    assert s[0, 0].item() == 1.0                                  # all-zero block
    assert torch.equal(q[:, :128].float(), torch.zeros(128, 128))
    assert s[0, 1].item() == pytest.approx(3 / 448)
    assert q[:, 128:].float().abs().max().item() == 448.0         # the block's largest magnitude maps to +-448
    # values above 448 * s (the scale of a block is fixed by its amax, so only an explicit grid shows the clamp): +-448
    big = torch.full((128, 128), 1e6)
    big[0, 0] = -1e6
    qb, sb = quantize_block128(big)
    assert qb.float().abs().max().item() == 448.0 and torch.isfinite(qb.float()).all()
    deq = dequantize_block128(qb, sb)
    assert deq.dtype == torch.bfloat16 and deq.shape == (128, 128)
    with pytest.raises(ValueError):
        quantize_block128(torch.zeros(100, 128))
    with pytest.raises(ValueError):
        dequantize_block128(q, s[:, :1])


# ---------------------------------------------------------------- C-ABI layer through the host simulation
_SO = build_sim.build()


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


def _create(lib, fmt=L.WEIGHTS_FP8_E4M3_B128, **kw):
    h = C.c_void_p()
    rc = lib.b2m_ctx_create_ex(C.byref(_cfg(**kw)), fmt, C.byref(h))
    return rc, h


def _stats(lib, h):
    s = L.Stats()
    assert lib.b2m_stats_get(h, C.byref(s)) == 0
    return s.as_dict()


def test_create_ex_accepts_and_refuses(sim):
    for kw in (dict(), dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, gate_dtype=L.DTYPE_F32),
               dict(hidden=4096, inter=14336, num_slots=2), dict(hidden=2048, inter=1408, num_slots=2, gemm_impl=2)):
        rc, h = _create(sim, **kw)
        assert rc == 0, (kw, sim.b2m_last_error(None))
        sim.b2m_ctx_destroy(h)
    rc, h = _create(sim, fmt=L.WEIGHTS_MODEL_DTYPE)       # format 0 = b2m_ctx_create
    assert rc == 0
    assert _stats(sim, h)["slot_bytes"] == 3 * 256 * 512 * 2
    sim.b2m_ctx_destroy(h)
    refused = [(dict(dtype=L.DTYPE_F16, gate_dtype=L.DTYPE_F16), L.B2M_EUNSUPPORTED, b"bf16"),
               (dict(dtype=L.DTYPE_F32), L.B2M_EUNSUPPORTED, b"bf16"),
               (dict(hidden=4104), L.B2M_EUNSUPPORTED, b"multiples of 128"),
               (dict(inter=520), L.B2M_EUNSUPPORTED, b"multiples of 128"),
               (dict(gemm_impl=1), L.B2M_EUNSUPPORTED, b"gemm_impl")]
    refused += [(dict(expert_type=t), L.B2M_EUNSUPPORTED, b"expert_type") for t in range(4)]
    for kw, code, msg in refused:
        rc, _ = _create(sim, **kw)
        assert rc == code, kw
        assert msg in sim.b2m_last_error(None), (kw, sim.b2m_last_error(None))
    for fmt in (-1, 2, 3):
        assert _create(sim, fmt=fmt)[0] == L.B2M_EINVAL
    # an fp8 MODEL dtype stays unsupported, whatever the weight format
    assert _create(sim, dtype=L.DTYPE_FP8)[0] == L.B2M_EUNSUPPORTED
    assert _create(sim, fmt=L.WEIGHTS_MODEL_DTYPE, dtype=L.DTYPE_FP8)[0] == L.B2M_EUNSUPPORTED


def test_slot_size_count_and_blob_checks(sim):
    H, I = 256, 512
    blob = expert_blob_bytes(H, I)
    assert blob == 3 * H * I + 3 * 2 * 4 * 4
    rc, h = _create(sim)
    assert rc == 0
    assert _stats(sim, h)["slot_bytes"] == blob
    bf16_blob = np.zeros(3 * H * I * 2, dtype=np.uint8)
    assert sim.b2m_register_expert(h, 0, 0, bf16_blob.ctypes.data, bf16_blob.nbytes) == L.B2M_EINVAL
    ok = np.zeros(blob, dtype=np.uint8)
    assert sim.b2m_register_expert(h, 0, 0, ok.ctypes.data, ok.nbytes) == 0
    # expert parallelism is refused on an fp8 context
    assert sim.b2m_ep_pack(h, 2, 0, 64, 8, None, None, None) == L.B2M_EUNSUPPORTED
    hd = (C.c_uint8 * 64)()
    assert sim.b2m_ep_p2p_init(h, 2, 0, 16, hd) == L.B2M_EUNSUPPORTED
    sim.b2m_ctx_destroy(h)
    # device_memory_ratio: about twice the bf16 slot count for the same budget (128 MiB for 12-MiB bf16 / 6-MiB fp8 experts)
    sim.b2m_sim_set_total_mem(256 << 20)
    try:
        counts = {}
        for fmt in (L.WEIGHTS_MODEL_DTYPE, L.WEIGHTS_FP8_E4M3_B128):
            rc, h = _create(sim, fmt=fmt, hidden=1024, inter=2048, num_layers=16, num_slots=0, device_memory_ratio=0.5)
            assert rc == 0, sim.b2m_last_error(None)
            counts[fmt] = _stats(sim, h)["slots"]
            sim.b2m_ctx_destroy(h)
        assert counts[L.WEIGHTS_MODEL_DTYPE] == 10 and counts[L.WEIGHTS_FP8_E4M3_B128] == 21
    finally:
        sim.b2m_sim_set_total_mem(TOTAL_MEM)


def test_offload_stages_fp8_sized_copies(sim):
    H, I, E = 256, 512, 8
    blob = expert_blob_bytes(H, I)
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
    # a resident slot holds exactly its expert's fp8 blob
    for e in range(E):
        if sim.b2m_is_resident(h, 1, e) == 1:
            p = C.c_void_p()
            assert sim.b2m_expert_dev_ptr(h, 1, e, C.byref(p)) == 0
            assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * blob).from_address(p.value)), blobs[1][e])
    sim.b2m_ctx_destroy(h)


def test_library_has_fp8_sass(lib_built):
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    fns = sass.split("Function : ")
    gemm = [f for f in fns if f.startswith("_ZN3b2m22grouped_gemm_tc_kernel")]
    fp8 = [f for f in gemm if "F2FP.F16.E4M3" in f]
    assert len(fp8) == 9, "one fp8 instantiation per tile width (gate/up 16..128, down 16..256)"
    for f in fp8:
        # register-A wgmma: HGMMA's A operand is a register, B a shared-memory descriptor
        assert any(ln.split("HGMMA", 1)[1].split(",")[1].strip().startswith("R") for ln in f.split("\n") if "HGMMA" in ln)
