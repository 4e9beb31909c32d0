"""CPU: int4 expert weights (B2M_WEIGHTS_INT4_G128, moe-infinity_b200/csrc/int4_weights.cuh and moe_infinity_b200/int4.py).

* the header's host dequantisation equals torch's (s.float() * (q.float() - z.float())).to(torch.bfloat16) bit for bit for
  every (q, z) pair, under scales of both signs from 2^-133 to 2^100, with normal and subnormal products and +-0;
* blob size, part offsets and the tile-major group grid against the header;
* quantize_g128 / dequantize_g128: round-trip bounds, exact round trip on the code grid, degenerate groups;
* b2m_ctx_create_ex through the host simulation of the C-ABI layer (tests/host/sim): accepted and refused configurations,
  slot size and count, blob size checks, expert parallelism refused, int4-sized staging copies;
* the built library holds nine int4 GEMM instantiations with register-A HGMMAs and bf16x2 dequantisation."""
from __future__ import annotations

import ctypes as C
import os
import re
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
from moe_infinity_b200.int4 import (dequantize_g128, expert_blob_bytes, pack_groups, quantize_g128,  # noqa: E402
                                    unpack_codes)

TOTAL_MEM = 8 << 30   # the simulation's default device memory


def _bf16_bits(x: float) -> int:
    return int(torch.tensor([x]).to(torch.bfloat16).view(torch.int16).item()) & 0xffff


# scale bit patterns: +-1, ordinary values, the smallest subnormal 2^-133 (+-), other subnormals, the smallest normal,
# 2^-120, values near 2^100 (+-), +-0
SCALES = [0x3f80, 0xbf80, _bf16_bits(0.0123), _bf16_bits(-3.7e5), 0x0001, 0x8001, 0x0007, 0x007f, 0x8043, 0x0080, 0x00ab,
          0x0380, 0x7180, 0xf1ff, 0x3c01, 0xbc7f, 0x0000, 0x8000]


def _host_check(tmp_path, *scales):
    exe = tmp_path / "int4_weights_check"
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "moe-infinity_b200", "csrc"),
                    os.path.join(HERE, "host", "int4_weights_check.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)] + ["%04x" % s for s in scales], capture_output=True, text=True, timeout=60, check=True)
    return r.stdout.strip().split("\n")


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_host_dequant_matches_torch(tmp_path):
    lines = _host_check(tmp_path, *SCALES)
    pairs = torch.arange(256)
    q, z = (pairs // 16).float(), (pairs % 16).float()
    seen_sub = seen_negzero = False
    for sb, line in zip(SCALES, lines):
        f = line.split()
        assert int(f[0], 16) == sb
        got = torch.tensor([int(v, 16) for v in f[1:]], dtype=torch.int32)
        s = torch.tensor([sb], dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
        want = (s * (q - z)).to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xffff
        assert torch.equal(got, want), f"scale {sb:04x}: pairs {(got != want).nonzero().flatten().tolist()[:8]}"
        seen_sub |= bool(((got & 0x7f80) == 0).logical_and((got & 0x7f) != 0).any())
        seen_negzero |= bool((got == 0x8000).any())
    assert seen_sub and seen_negzero, "the scales reach bf16 subnormal products and -0"


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_layout_matches_header(tmp_path):
    tail = dict(ln.split(" ", 1) for ln in _host_check(tmp_path))
    assert tail["blob"].split() == [str(expert_blob_bytes(4096, 14336)), str(expert_blob_bytes(2048, 1408)),
                                    str(expert_blob_bytes(6144, 16384))]
    assert tail["blob"].split()[0] == "93585408"
    assert 56 * 8 * expert_blob_bytes(6144, 16384) < 72e9          # Mixtral-8x22B's routed experts fit in 80 GB
    m, g = 2048 * 1408 // 2, 2048 * 1408 // 128 * 4
    assert tail["parts"].split() == [str(v) for mm in range(3) for v in (mm * m, 3 * m + mm * g)]
    # pack_groups puts (r, g) where the header's grid_index says: encode r and g in the word itself
    rows, cols = 384, 512
    r = torch.arange(rows)[:, None].expand(rows, cols // 128)
    gg = torch.arange(cols // 128)[None, :].expand(rows, cols // 128)
    s = (r * 4 + gg).to(torch.int16).view(torch.bfloat16)
    z = (gg * 3 % 16).to(torch.uint8)
    words = pack_groups(s, z).view(torch.int32)
    idx = [int(v) for v in tail["grid"].split()]
    for (rr, g_), i in zip([(0, 0), (1, 0), (127, 0), (0, 1), (127, 3), (128, 0), (200, 2), (383, 3)], idx):
        assert int(words[i]) == (rr * 4 + g_) | ((g_ * 3 % 16) << 16)
    assert tail["tile"] == "ok"


def test_quantize_roundtrip_bounds():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(256, 384, generator=g) * 0.02
    w[:128, 128:256] *= 1000                                       # groups of very different ranges
    w[200, :128] = torch.linspace(-5, 3, 128)
    q, s, z = quantize_g128(w)
    assert q.shape == (256, 192) and q.dtype == torch.uint8
    assert s.shape == (256, 3) and s.dtype == torch.bfloat16 and z.shape == (256, 3) and z.dtype == torch.uint8
    assert int(z.max()) <= 15
    deq = dequantize_g128(q, s, z, torch.float32)
    se = s.float().repeat_interleave(128, 1)
    # round to nearest: half a step, plus what the bf16 rounding of s and of W add
    assert bool(((deq - w).abs() <= 0.6 * se.abs() + w.abs() * 2.0 ** -7).all())
    # min and max of each group are reached within half a step
    b = w.reshape(256, 3, 128)
    d = deq.reshape(256, 3, 128)
    assert bool(((d.amin(2) - b.amin(2)).abs() <= 0.6 * s.float()).all())
    assert bool(((d.amax(2) - b.amax(2)).abs() <= 0.6 * s.float() + b.amax(2).abs() * 2.0 ** -7).all())


def test_quantize_exact_on_grid():
    """Weights that are exactly s * (q - z) with both ends of the code range present come back bit for bit."""
    g = torch.Generator().manual_seed(1)
    rows, cols = 128, 256
    codes = torch.randint(0, 16, (rows, cols), generator=g, dtype=torch.uint8)
    codes[:, ::128] = 0
    codes[:, 1::128] = 15
    z = torch.randint(0, 16, (rows, cols // 128), generator=g, dtype=torch.uint8)
    s = torch.exp2(torch.randint(-20, 5, (rows, cols // 128), generator=g).float()).to(torch.bfloat16)
    q = codes[:, 0::2] | (codes[:, 1::2] << 4)
    w = dequantize_g128(q, s, z, torch.float32)
    q2, s2, z2 = quantize_g128(w)
    assert torch.equal(s2, s) and torch.equal(z2, z) and torch.equal(q2, q)
    assert torch.equal(unpack_codes(q2), codes)


def test_degenerate_groups():
    w = torch.zeros(128, 512)
    w[:, 128:256] = 0.7                                            # all-equal
    w[:, 256:384] = -3.25
    w[:, 384:] = torch.randn(128, 128)
    q, s, z = quantize_g128(w)
    codes = unpack_codes(q)
    assert bool((s[:, 0].float() == 1).all()) and bool((z[:, 0] == 0).all()) and bool((codes[:, :128] == 0).all())
    assert bool((s[:, 1] == torch.tensor(0.7).to(torch.bfloat16)).all()) and bool((z[:, 1] == 0).all())
    assert bool((codes[:, 128:384] == 1).all())
    deq = dequantize_g128(q, s, z)
    assert bool((deq[:, :128] == 0).all())
    assert bool((deq[:, 128:256] == torch.tensor(0.7).to(torch.bfloat16)).all())
    assert bool((deq[:, 256:384].float() == -3.25).all())
    with pytest.raises(ValueError):
        quantize_g128(torch.zeros(128, 100))
    with pytest.raises(ValueError):
        dequantize_g128(q, s[:, :1], z)
    with pytest.raises(ValueError):
        dequantize_g128(q, s.float(), z)


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


def _create(lib, fmt=L.WEIGHTS_INT4_G128, **kw):
    h = C.c_void_p()
    rc = lib.b2m_ctx_create_ex(C.byref(_cfg(**kw)), fmt, C.byref(h))
    return rc, h


def _stats(lib, h):
    s = L.Stats()
    assert lib.b2m_stats_get(h, C.byref(s)) == 0
    return s.as_dict()


def test_create_ex_int4_accepts_and_refuses(sim):
    assert L.WEIGHTS_INT4_G128 == 4
    for kw in (dict(), dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, gate_dtype=L.DTYPE_F32),
               dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_V3, gate_dtype=L.DTYPE_F32, num_experts=16,
                    top_k=4, n_group=4, topk_group=2, shared_inter=256),
               dict(hidden=4096, inter=14336, num_slots=2), dict(hidden=2048, inter=1408, num_slots=2, gemm_impl=2)):
        rc, h = _create(sim, **kw)
        assert rc == 0, (kw, sim.b2m_last_error(None))
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
        err = sim.b2m_last_error(None)
        assert msg in err and b"int4" in err, (kw, err)
    for fmt in (-1, 2, 3, 5):                                         # 2 and 3 are not weight formats
        assert _create(sim, fmt=fmt)[0] == L.B2M_EINVAL


def test_int4_slot_size_count_and_blob_checks(sim):
    H, I = 256, 512
    blob = expert_blob_bytes(H, I)
    assert blob == 3 * H * I // 2 + 3 * (H * I // 128) * 4
    rc, h = _create(sim)
    assert rc == 0
    assert _stats(sim, h)["slot_bytes"] == blob
    for wrong in (3 * H * I * 2, 3 * H * I + 3 * 2 * 4 * 4, blob - 4, blob + 16):   # bf16, fp8, short, long
        b = np.zeros(wrong, dtype=np.uint8)
        assert sim.b2m_register_expert(h, 0, 0, b.ctypes.data, b.nbytes) == L.B2M_EINVAL, wrong
    ok = np.zeros(blob, dtype=np.uint8)
    assert sim.b2m_register_expert(h, 0, 0, ok.ctypes.data, ok.nbytes) == 0
    # expert parallelism is refused on an int4 context
    assert sim.b2m_ep_pack(h, 2, 0, 64, 8, None, None, None) == L.B2M_EUNSUPPORTED
    assert b"int4" in sim.b2m_last_error(h)
    hd = (C.c_uint8 * 64)()
    assert sim.b2m_ep_p2p_init(h, 2, 0, 16, hd) == L.B2M_EUNSUPPORTED
    sim.b2m_ctx_destroy(h)
    # device_memory_ratio: a 128 MiB budget holds 10 bf16, 21 fp8 and 40 int4 experts of H=1024, I=2048
    sim.b2m_sim_set_total_mem(256 << 20)
    try:
        counts = {}
        for fmt in (L.WEIGHTS_MODEL_DTYPE, L.WEIGHTS_FP8_E4M3_B128, L.WEIGHTS_INT4_G128):
            rc, h = _create(sim, fmt=fmt, hidden=1024, inter=2048, num_layers=16, num_slots=0, device_memory_ratio=0.5)
            assert rc == 0, sim.b2m_last_error(None)
            st = _stats(sim, h)
            counts[fmt] = st["slots"]
            if fmt == L.WEIGHTS_INT4_G128:
                assert st["slot_bytes"] == expert_blob_bytes(1024, 2048) == 3342336
            sim.b2m_ctx_destroy(h)
        assert counts == {L.WEIGHTS_MODEL_DTYPE: 10, L.WEIGHTS_FP8_E4M3_B128: 21, L.WEIGHTS_INT4_G128: 40}
    finally:
        sim.b2m_sim_set_total_mem(TOTAL_MEM)


def test_offload_stages_int4_sized_copies(sim):
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
    # a resident slot holds exactly its expert's int4 blob
    for e in range(E):
        if sim.b2m_is_resident(h, 1, e) == 1:
            p = C.c_void_p()
            assert sim.b2m_expert_dev_ptr(h, 1, e, C.byref(p)) == 0
            assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * blob).from_address(p.value)), blobs[1][e])
    sim.b2m_ctx_destroy(h)


def test_library_has_int4_sass(lib_built):
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    fns = sass.split("Function : ")
    # grouped_gemm_tc_kernel<NT, DUAL, DT_BF16, MC = 1, AS_INT4 = 3>
    pat = re.compile(r"_ZN3b2m22grouped_gemm_tc_kernelILi(\d+)ELb([01])ELi0ELi1ELi3EEEv")
    found = {}
    for f in fns:
        m = pat.match(f)
        if m:
            found[(int(m.group(1)), m.group(2) == "1")] = f
    assert sorted(found) == sorted([(n, True) for n in (16, 32, 64, 128)] + [(n, False) for n in (16, 32, 64, 128, 256)])
    for key, f in found.items():
        # register-A wgmma: HGMMA's A operand is a register, B a shared-memory descriptor
        assert any(ln.split("HGMMA", 1)[1].split(",")[1].strip().startswith("R") for ln in f.split("\n") if "HGMMA" in ln), key
        assert "HMUL2.BF16_V2" in f and ("HADD2.BF16_V2" in f or "HFMA2.BF16_V2" in f), key   # bf16x2 dequantisation
        assert "F2FP.F16.E4M3" not in f, key
