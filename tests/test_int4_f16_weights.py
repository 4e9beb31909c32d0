"""CPU: int4 expert weights with fp16 scales and f16 activations (B2M_WEIGHTS_INT4_G128_F16, the AWQ / GPTQ format).

* the header's host f16 dequantisation equals torch's (s.float() * (q.float() - z.float())).to(torch.float16) bit for bit
  for every (q, z) pair, under fp16 scales of both signs from the smallest subnormal to 65504 (subnormal products, +-0,
  overflow to +-Inf);
* int4.from_awq / int4.from_gptq (v1 and v2) against test-side packers: exact round trip, the dequantised matrix equal to
  AWQ's / GPTQ's own fp16 (q - z) * s, and their refusals; quantize_g128(scale_dtype=float16), f16 pack_groups;
* hf.load_int4_checkpoint on synthetic safetensors shards: every tensor reaches the engine, and the refusals;
* b2m_ctx_create_ex(format 6) through the host simulation: accepted and refused configurations, slot size equal to format 4,
  int4-sized offload staging, expert parallelism refused;
* the built library holds nine f16 int4 GEMM instantiations with register-A f16 HGMMAs and f16x2 dequantisation."""
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
sys.path.insert(0, HERE)

import build_sim  # noqa: E402
import int4_checkpoint_packers as P  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from moe_infinity_b200 import hf  # noqa: E402
from moe_infinity_b200.int4 import (dequantize_g128, expert_blob_bytes, from_awq, from_gptq, pack_groups,  # noqa: E402
                                    quantize_g128, unpack_codes)

TOTAL_MEM = 8 << 30   # the simulation's default device memory


def _f16_bits(x: float) -> int:
    return int(torch.tensor([x]).to(torch.float16).view(torch.int16).item()) & 0xffff


# fp16 scale bit patterns: +-1, ordinary values, the smallest subnormal 2^-24 (+-), other subnormals, the largest subnormal,
# the smallest normal, values whose products round, 2^15 and 65504 (+-: products overflow to +-Inf), +-0
SCALES = [0x3c00, 0xbc00, _f16_bits(0.0123), _f16_bits(-37.7), 0x0001, 0x8001, 0x0007, 0x02ab, 0x83ff, 0x0400, 0x0401,
          0x3c01, 0xb7ff, 0x1234, 0x5555, 0x7800, 0x7bff, 0xfbff, 0x0000, 0x8000]


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_host_f16_dequant_matches_torch(tmp_path):
    exe = tmp_path / "int4_f16_check"
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "moe-infinity_b200", "csrc"),
                    os.path.join(HERE, "host", "int4_f16_check.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)] + ["%04x" % s for s in SCALES], capture_output=True, text=True, timeout=60, check=True)
    lines = r.stdout.strip().split("\n")
    assert len(lines) == len(SCALES)
    pairs = torch.arange(256)
    q, z = (pairs // 16).float(), (pairs % 16).float()
    seen = dict(sub=False, negzero=False, inf=False, neginf=False)
    for sb, line in zip(SCALES, lines):
        f = line.split()
        assert int(f[0], 16) == sb
        got = torch.tensor([int(v, 16) for v in f[1:]], dtype=torch.int32)
        s = torch.tensor([sb], dtype=torch.int32).to(torch.int16).view(torch.float16).float()
        want = (s * (q - z)).to(torch.float16).view(torch.int16).to(torch.int32) & 0xffff
        assert torch.equal(got, want), f"scale {sb:04x}: pairs {(got != want).nonzero().flatten().tolist()[:8]}"
        seen["sub"] |= bool(((got & 0x7c00) == 0).logical_and((got & 0x3ff) != 0).any())
        seen["negzero"] |= bool((got == 0x8000).any())
        seen["inf"] |= bool((got == 0x7c00).any())
        seen["neginf"] |= bool((got == 0xfc00).any())
    assert all(seen.values()), seen


def test_quantize_f16_scales():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(256, 384, generator=g) * 0.02
    w[:128, 128:256] *= 1000
    q, s, z = quantize_g128(w, scale_dtype=torch.float16)
    assert s.dtype == torch.float16 and s.shape == (256, 3) and q.shape == (256, 192)
    deq = dequantize_g128(q, s, z, torch.float32)
    se = s.float().repeat_interleave(128, 1)
    assert bool(((deq - w).abs() <= 0.6 * se.abs() + w.abs() * 2.0 ** -10).all())
    # the default is the bf16 quantiser, unchanged
    qb, sb, zb = quantize_g128(w)
    q2, s2, z2 = quantize_g128(w, scale_dtype=torch.bfloat16)
    assert sb.dtype == torch.bfloat16 and torch.equal(qb, q2) and torch.equal(sb, s2) and torch.equal(zb, z2)
    # weights exactly on an fp16 grid come back bit for bit
    codes = torch.randint(0, 16, (128, 256), generator=g, dtype=torch.uint8)
    codes[:, ::128], codes[:, 1::128] = 0, 15
    zz = torch.randint(0, 16, (128, 2), generator=g, dtype=torch.uint8)
    ss = (torch.rand(128, 2, generator=g) * 2 + 0.5).to(torch.float16)
    qq = codes[:, 0::2] | (codes[:, 1::2] << 4)
    q3, s3, z3 = quantize_g128(dequantize_g128(qq, ss, zz, torch.float32), scale_dtype=torch.float16)
    assert torch.equal(s3, ss) and torch.equal(z3, zz) and torch.equal(q3, qq)
    with pytest.raises(ValueError):
        quantize_g128(w, scale_dtype=torch.float32)
    with pytest.raises(ValueError):
        quantize_g128(torch.linspace(-1e6, 1e6, 128).repeat(128, 1), scale_dtype=torch.float16)   # scale overflows fp16


def test_pack_groups_f16():
    s = (torch.arange(256 * 2).reshape(256, 2) * 0.01 - 1).to(torch.float16)
    z = (torch.arange(256 * 2).reshape(256, 2) % 16).to(torch.uint8)
    words = pack_groups(s, z).view(torch.int32)
    bits = s.view(torch.int16).to(torch.int32) & 0xffff
    for r, g in [(0, 0), (5, 1), (127, 1), (128, 0), (255, 1)]:
        assert int(words[((r // 128) * 2 + g) * 128 + r % 128]) == int(bits[r, g]) | (int(z[r, g]) << 16)


@pytest.mark.parametrize("fmt", ["awq", "gptq", "gptq_v2"])
def test_checkpoint_unpack_roundtrip(fmt):
    g = torch.Generator().manual_seed(["awq", "gptq", "gptq_v2"].index(fmt))
    out, n_in = 256, 384
    q, s, z = P.random_qsz(out, n_in, g, z_lo=1 if fmt == "gptq" else 0)
    s[0, 0] = -s[0, 0].abs() - 0.01                        # a negative scale, a subnormal one, and large ones
    s[1, 1] = torch.tensor(3e-7, dtype=torch.float16)
    s[2, :] = torch.tensor(4000.0, dtype=torch.float16)
    if fmt == "awq":
        q2, s2, z2 = from_awq(*P.awq_pack(q, s, z))
    else:
        q2, s2, z2 = from_gptq(*P.gptq_pack(q, s, z, v1=fmt == "gptq"), checkpoint_format=fmt)
    assert q2.dtype == torch.uint8 and q2.shape == (out, n_in // 2)
    assert torch.equal(unpack_codes(q2).long(), q)
    assert s2.dtype == torch.float16 and torch.equal(s2.view(torch.int16), s.view(torch.int16))
    assert z2.dtype == torch.uint8 and torch.equal(z2.long(), z)
    want = P.fp16_dequant(q, s, z)
    got = dequantize_g128(q2, s2, z2, torch.float16)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_checkpoint_unpack_refusals():
    g = torch.Generator().manual_seed(9)
    q, s, z = P.random_qsz(128, 256, g, z_lo=1)
    qw, qz, sc = P.awq_pack(q, s, z)
    with pytest.raises(ValueError, match="group size"):
        from_awq(qw, qz, torch.cat([sc, sc]))               # 64-input groups
    with pytest.raises(ValueError, match="int32"):
        from_awq(qw.to(torch.int64), qz, sc)
    with pytest.raises(ValueError, match="float16"):
        from_awq(qw, qz, sc.to(torch.bfloat16))
    gw, gz, gs, gi = P.gptq_pack(q, s, z)
    with pytest.raises(ValueError, match="group size"):
        from_gptq(gw, gz, torch.cat([gs, gs]), gi)
    with pytest.raises(ValueError, match="act-order"):
        from_gptq(gw, gz, gs, gi.flip(0))
    with pytest.raises(ValueError, match="checkpoint_format"):
        from_gptq(gw, gz, gs, gi, checkpoint_format="marlin")
    z16 = z.clone()
    z16[3, 1] = 16                                          # a v1 zero point of 16 is stored as 15
    gw, gz, gs, gi = P.gptq_pack(q, s, z16)
    with pytest.raises(ValueError, match="qzeros"):
        from_gptq(gw, gz, gs, gi)
    # the same stored bits are z = 15 for a v2 checkpoint
    _, _, z2 = from_gptq(gw, gz, gs, gi, checkpoint_format="gptq_v2")
    assert int(z2[3, 1]) == 15


# ---------------------------------------------------------------- hf.load_int4_checkpoint on synthetic shards
class _FakeEngine:
    """Records what load_int4_checkpoint hands an engine (the real one needs a GPU)."""

    def __init__(self, L_, E, H, I, expert_type, shared_inter=0, router=L.ROUTER_MIXTRAL, dtype=torch.float16):
        self.int4, self.dtype = True, dtype
        self.L, self.E, self.H, self.I = L_, E, H, I
        self.expert_type, self.shared_inter, self.router = expert_type, shared_inter, router
        self.experts, self.shared, self.gates, self.biases, self.resident = {}, {}, {}, {}, {}

    def load_expert(self, l, e, qs, scales=None, zeros=None):
        self.experts[(l, e)] = (qs, scales, zeros)
        self.resident[(l, e)] = True

    def register_expert(self, l, e, qs, scales=None, zeros=None):
        self.experts[(l, e)] = (qs, scales, zeros)
        self.resident[(l, e)] = False

    def register_shared(self, l, ws):
        self.shared[l] = ws

    def set_gate(self, l, w):
        self.gates[l] = w

    def set_gate_bias(self, l, b):
        self.biases[l] = b


def _mixtral_checkpoint(tmp_path, method, L_=2, E=4, H=256, I=384, seed=0):
    g = torch.Generator().manual_seed(seed)
    tensors, truth = {}, {}
    for l in range(L_):
        base = f"model.layers.{l}.block_sparse_moe"
        tensors[f"{base}.gate.weight"] = torch.randn(E, H, generator=g).to(torch.float16)
        for e in range(E):
            for n, (o, i) in zip(("w1", "w2", "w3"), ((I, H), (H, I), (I, H))):
                q, s, z = P.random_qsz(o, i, g, z_lo=1)
                truth[(l, e, n)] = (q, s, z)
                pre = f"{base}.experts.{e}.{n}"
                if method == "awq":
                    qw, qz, sc = P.awq_pack(q, s, z)
                    tensors.update({f"{pre}.qweight": qw, f"{pre}.qzeros": qz, f"{pre}.scales": sc})
                else:
                    qw, qz, sc, gi = P.gptq_pack(q, s, z)
                    tensors.update({f"{pre}.qweight": qw, f"{pre}.qzeros": qz, f"{pre}.scales": sc, f"{pre}.g_idx": gi})
    return tensors, truth


AWQ_CFG = dict(quant_method="awq", bits=4, group_size=128, zero_point=True, version="gemm")
GPTQ_CFG = dict(quant_method="gptq", bits=4, group_size=128, desc_act=False, sym=False, checkpoint_format="gptq")


@pytest.mark.parametrize("method", ["awq", "gptq"])
def test_load_int4_checkpoint_mixtral(tmp_path, method):
    tensors, truth = _mixtral_checkpoint(tmp_path, method)
    shards = P.write_shards(str(tmp_path), tensors)
    eng = _FakeEngine(2, 4, 256, 384, L.EXPERT_MIXTRAL)
    cfg = AWQ_CFG if method == "awq" else GPTQ_CFG
    assert hf.load_int4_checkpoint(eng, shards, cfg, "mixtral", resident=False) == [0, 1]
    assert sorted(eng.experts) == [(l, e) for l in range(2) for e in range(4)] and not any(eng.resident.values())
    for (l, e), (qs, ss, zs) in eng.experts.items():
        for n, q2, s2, z2 in zip(("w1", "w2", "w3"), qs, ss, zs):
            q, s, z = truth[(l, e, n)]
            assert torch.equal(unpack_codes(q2).long(), q) and torch.equal(s2, s) and torch.equal(z2.long(), z)
    for l in range(2):
        assert torch.equal(eng.gates[l], tensors[f"model.layers.{l}.block_sparse_moe.gate.weight"])


def test_load_int4_checkpoint_deepseek(tmp_path):
    """GPTQ v2, a dense first layer (skipped), quantised shared experts (dequantised to f16) and a V3 correction bias."""
    g = torch.Generator().manual_seed(3)
    H, I, Is, E = 256, 128, 256, 4
    tensors, truth = {"model.layers.0.mlp.gate_proj.weight": torch.zeros(4, 4, dtype=torch.float16)}, {}
    base = "model.layers.1.mlp"
    tensors[f"{base}.gate.weight"] = torch.randn(E, H, generator=g)
    tensors[f"{base}.gate.e_score_correction_bias"] = torch.randn(E, generator=g)

    def put(pre, o, i):
        q, s, z = P.random_qsz(o, i, g)
        qw, qz, sc, _ = P.gptq_pack(q, s, z, v1=False)
        tensors.update({f"{pre}.qweight": qw, f"{pre}.qzeros": qz, f"{pre}.scales": sc})
        truth[pre] = (q, s, z)

    names = ("gate_proj", "up_proj", "down_proj")
    for e in range(E):
        for n, (o, i) in zip(names, ((I, H), (I, H), (H, I))):
            put(f"{base}.experts.{e}.{n}", o, i)
    for n, (o, i) in zip(names, ((Is, H), (Is, H), (H, Is))):
        put(f"{base}.shared_experts.{n}", o, i)
    shards = P.write_shards(str(tmp_path), tensors, nshards=3)
    eng = _FakeEngine(2, E, H, I, L.EXPERT_DEEPSEEK, shared_inter=Is, router=L.ROUTER_DEEPSEEK_V3)
    cfg = dict(GPTQ_CFG, checkpoint_format="gptq_v2")
    assert hf.load_int4_checkpoint(eng, shards, cfg, "deepseek_v3") == [1]
    assert sorted(eng.experts) == [(1, e) for e in range(E)] and all(eng.resident.values())
    for e in range(E):
        for n, q2, s2, z2 in zip(names, *eng.experts[(1, e)]):
            q, s, z = truth[f"{base}.experts.{e}.{n}"]
            assert torch.equal(unpack_codes(q2).long(), q) and torch.equal(s2, s) and torch.equal(z2.long(), z)
    for n, w in zip(names, eng.shared[1]):
        assert w.dtype == torch.float16 and torch.equal(w, P.fp16_dequant(*truth[f"{base}.shared_experts.{n}"]))
    assert torch.equal(eng.gates[1], tensors[f"{base}.gate.weight"])
    assert torch.equal(eng.biases[1], tensors[f"{base}.gate.e_score_correction_bias"])


def test_load_int4_checkpoint_refusals(tmp_path):
    tensors, _ = _mixtral_checkpoint(tmp_path, "gptq", L_=1, E=2)
    shards = P.write_shards(str(tmp_path), tensors)
    eng = _FakeEngine(1, 2, 256, 384, L.EXPERT_MIXTRAL)
    for cfg, msg in ((dict(GPTQ_CFG, bits=8), "bits"), (dict(GPTQ_CFG, group_size=64), "group_size"),
                     (dict(AWQ_CFG, zero_point=False), "zero_point"), (dict(AWQ_CFG, version="gemv"), "gemm"),
                     (dict(GPTQ_CFG, checkpoint_format="marlin"), "checkpoint_format"),
                     (dict(quant_method="bitsandbytes", bits=4, group_size=128), "quant_method")):
        with pytest.raises(ValueError, match=msg):
            hf.load_int4_checkpoint(eng, shards, cfg, "mixtral")
    with pytest.raises(ValueError, match="float16"):
        hf.load_int4_checkpoint(_FakeEngine(1, 2, 256, 384, L.EXPERT_MIXTRAL, dtype=torch.bfloat16), shards, GPTQ_CFG, "mixtral")
    # act-order: a g_idx other than c // 128
    bad = dict(tensors)
    key = "model.layers.0.block_sparse_moe.experts.1.w2.g_idx"
    bad[key] = bad[key].flip(0).contiguous()
    d = tmp_path / "actorder"
    d.mkdir()
    with pytest.raises(ValueError, match="act-order"):
        hf.load_int4_checkpoint(eng, P.write_shards(str(d), bad), dict(GPTQ_CFG, desc_act=True), "mixtral")
    # a missing tensor is named (the first one in load order)
    short = {k: v for k, v in tensors.items() if ".experts.1.w3." not in k}
    d = tmp_path / "missing"
    d.mkdir()
    with pytest.raises(ValueError, match=re.escape("model.layers.0.block_sparse_moe.experts.1.w3.qweight")):
        hf.load_int4_checkpoint(eng, P.write_shards(str(d), short), GPTQ_CFG, "mixtral")


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
    cfg.dtype, cfg.expert_type, cfg.router, cfg.max_tokens = L.DTYPE_F16, L.EXPERT_MIXTRAL, L.ROUTER_MIXTRAL, 64
    cfg.gate_dtype = L.DTYPE_F16
    cfg.routed_scaling_factor = 1.0
    cfg.num_slots = 16
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _create(lib, fmt=L.WEIGHTS_INT4_G128_F16, **kw):
    h = C.c_void_p()
    rc = lib.b2m_ctx_create_ex(C.byref(_cfg(**kw)), fmt, C.byref(h))
    return rc, h


def _stats(lib, h):
    s = L.Stats()
    assert lib.b2m_stats_get(h, C.byref(s)) == 0
    return s.as_dict()


def test_create_ex_int4_f16_accepts_and_refuses(sim):
    assert L.WEIGHTS_INT4_G128_F16 == 6
    for kw in (dict(), dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GREEDY, gate_dtype=L.DTYPE_F32),
               dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_V3, gate_dtype=L.DTYPE_F32, num_experts=16,
                    top_k=4, n_group=4, topk_group=2, shared_inter=256),
               dict(hidden=4096, inter=14336, num_slots=2), dict(hidden=2048, inter=1408, num_slots=2, gemm_impl=2)):
        rc, h = _create(sim, **kw)
        assert rc == 0, (kw, sim.b2m_last_error(None))
        sim.b2m_ctx_destroy(h)
    refused = [(dict(dtype=L.DTYPE_BF16, gate_dtype=L.DTYPE_BF16), b"f16"),
               (dict(dtype=L.DTYPE_F32), b"f16"),
               (dict(hidden=4104), b"multiples of 128"),
               (dict(inter=520), b"multiples of 128"),
               (dict(gemm_impl=1), b"gemm_impl")]
    refused += [(dict(expert_type=t), b"expert_type") for t in range(4)]
    for kw, msg in refused:
        rc, _ = _create(sim, **kw)
        assert rc == L.B2M_EUNSUPPORTED, kw
        err = sim.b2m_last_error(None)
        assert msg in err and b"int4" in err, (kw, err)
    assert _create(sim, fmt=5)[0] == L.B2M_EINVAL


def test_int4_f16_slot_size_and_ep_refused(sim):
    H, I = 256, 512
    blob = expert_blob_bytes(H, I)
    rc, h = _create(sim)
    assert rc == 0
    assert _stats(sim, h)["slot_bytes"] == blob
    rc4, h4 = _create(sim, fmt=L.WEIGHTS_INT4_G128, dtype=L.DTYPE_BF16, gate_dtype=L.DTYPE_BF16)
    assert rc4 == 0 and _stats(sim, h4)["slot_bytes"] == blob
    sim.b2m_ctx_destroy(h4)
    for wrong in (3 * H * I * 2, blob - 4, blob + 16):
        b = np.zeros(wrong, dtype=np.uint8)
        assert sim.b2m_register_expert(h, 0, 0, b.ctypes.data, b.nbytes) == L.B2M_EINVAL, wrong
    assert sim.b2m_ep_pack(h, 2, 0, 64, 8, None, None, None) == L.B2M_EUNSUPPORTED
    assert b"int4" in sim.b2m_last_error(h)
    hd = (C.c_uint8 * 64)()
    assert sim.b2m_ep_p2p_init(h, 2, 0, 16, hd) == L.B2M_EUNSUPPORTED
    sim.b2m_ctx_destroy(h)
    # a Mixtral-8x7B expert takes the same 93 585 408 B in both int4 formats
    rc, h = _create(sim, hidden=4096, inter=14336, num_slots=2)
    assert rc == 0 and _stats(sim, h)["slot_bytes"] == 93585408
    sim.b2m_ctx_destroy(h)


def test_offload_stages_int4_f16_sized_copies(sim):
    H, I, E = 256, 512, 8
    blob = expert_blob_bytes(H, I)
    rc, h = _create(sim, num_slots=3)
    assert rc == 0
    rng = np.random.default_rng(1)
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
    assert staged >= st["misses"] * blob and staged < st["misses"] * blob + 4096
    for e in range(E):
        if sim.b2m_is_resident(h, 1, e) == 1:
            p = C.c_void_p()
            assert sim.b2m_expert_dev_ptr(h, 1, e, C.byref(p)) == 0
            assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * blob).from_address(p.value)), blobs[1][e])
    sim.b2m_ctx_destroy(h)


def test_library_has_int4_f16_sass(lib_built):
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    fns = sass.split("Function : ")
    # grouped_gemm_tc_kernel<NT, DUAL, DT_F16 = 2, MC = 1, AS_INT4 = 3>
    pat = re.compile(r"_ZN3b2m22grouped_gemm_tc_kernelILi(\d+)ELb([01])ELi2ELi1ELi3EEEv")
    found = {}
    for f in fns:
        m = pat.match(f)
        if m:
            found[(int(m.group(1)), m.group(2) == "1")] = f
    assert sorted(found) == sorted([(n, True) for n in (16, 32, 64, 128)] + [(n, False) for n in (16, 32, 64, 128, 256)])
    for key, f in found.items():
        lines = f.split("\n")
        hg = [ln for ln in lines if "HGMMA" in ln]
        # register-A wgmma with f16 operands (SASS names only the bf16 variant: HGMMA.64xNx16.F32.BF16)
        assert any(ln.split("HGMMA", 1)[1].split(",")[1].strip().startswith("R") for ln in hg), key
        assert hg and not any(".BF16" in ln for ln in hg), key
        assert any(re.search(r"\bHMUL2 ", ln) for ln in lines), key                                  # f16x2 * s
        assert any(re.search(r"\bH(ADD|FMA)2 ", ln) for ln in lines), key                            # f16x2 q - z
        assert "BF16_V2" not in f, key
        assert "F2FP.F16.E4M3" not in f, key
