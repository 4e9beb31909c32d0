"""CPU: the rows of tests/gemm_exact_cases.py run the launch plans they claim, together cover every plan and A source of the
grouped expert GEMMs, and their float64 reference is oracle.expert_ffn bit for bit.

* Plans: each row's routing and expert launches go through the host simulation of api.cu (tests/host/sim, as in
  test_host_sim.py), on 132 simulated SMs with the default switches; the logged K3 / K4 launches must show the row's token-tile
  widths, split-K / stream-K, dual_m and early-A flags, and for stream-K rows the largest number of CTAs one tile spans under
  gemm_body's partition (CTA b takes units [units * b / 132, units * (b + 1) / 132)).
* Coverage: the union of the rows holds every tile width, split-K plan, dual_m case, ragged shape, A source, expert type,
  numerics mode and the offload waves that tests/test_gpu_gemm_exact.py then checks exactly on the GPU.
* Reference: at small sizes the reference equals oracle.expert_ffn, which tests/test_oracle_expert_ref.py pins to the
  reference's own compiled expert modules."""
from __future__ import annotations

import ctypes as C
import os
import re
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host", "sim"))

import build_sim  # noqa: E402
import gemm_exact_cases as X  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from oracle import moe_oracle as O  # noqa: E402

_SO = build_sim.build()


# ------------------------------------------------------------------------------------------------ plans
@pytest.fixture(scope="module")
def sim():
    if _SO is None:
        pytest.skip("nvcc / g++ not available to build the host simulation")
    lib = C.CDLL(_SO)
    for name, res, args in L.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    lib.b2m_sim_take_log.restype, lib.b2m_sim_take_log.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t]
    return lib


def _take_log(lib):
    buf = C.create_string_buffer(1 << 22)
    assert lib.b2m_sim_take_log(buf, len(buf)) < len(buf)
    return [ln for ln in buf.value.decode().split("\n") if ln]


def _kv(line):
    return {m.group(1): m.group(2) for m in re.finditer(r"(\w+)=(\[[^\]]*\]|\S+)", line)}


_DT = {"bf16": L.DTYPE_BF16, "f16": L.DTYPE_F16, "f32": L.DTYPE_F32}


class SimEngine:
    """One simulated context for the rows sharing an engine key: zero-filled host blobs stand in for the weights (the
    planner never reads them)."""

    def __init__(self, lib, c: X.Case, max_tokens: int):
        self.lib, self.c = lib, c
        cfg = L.Config()
        cfg.struct_size = C.sizeof(L.Config)
        cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = 1, c.E, c.H, c.I, c.k
        cfg.dtype, cfg.expert_type, cfg.max_tokens = _DT[c.dtype], X.ETYPE[c.etype], max_tokens
        deepseek = c.etype == X.DEEPSEEK
        cfg.router = L.ROUTER_DEEPSEEK_GREEDY if deepseek else L.ROUTER_MIXTRAL
        cfg.gate_dtype = L.DTYPE_F32 if deepseek else _DT[c.dtype]
        cfg.numerics = L.NUMERICS_FP32 if c.numerics == "fp32" else L.NUMERICS_REFERENCE
        cfg.num_slots = c.slots or c.E
        cfg.shared_inter = c.shared
        cfg.gemm_impl = c.gemm_impl if c.gemm_impl else (0 if c.fmt == "pk12" else 2)
        cfg.device_memory_ratio = 0.5
        cfg.routed_scaling_factor = 1.0
        self.h = C.c_void_p()
        assert lib.b2m_ctx_create(C.byref(cfg), C.byref(self.h)) == 0, self.err()
        s = L.Stats()
        assert lib.b2m_stats_get(self.h, C.byref(s)) == 0
        self.blob = np.zeros(s.as_dict()["slot_bytes"], dtype=np.uint8)
        for e in range(c.E):
            assert lib.b2m_register_expert(self.h, 0, e, self.blob.ctypes.data, self.blob.nbytes) == 0, self.err()
        if c.shared:
            es = 4 if c.dtype == "f32" else 2
            self.shared = np.zeros(3 * c.H * c.shared * es, dtype=np.uint8)
            assert lib.b2m_register_shared(self.h, 0, self.shared.ctypes.data, self.shared.nbytes) == 0, self.err()

    def err(self):
        return (self.lib.b2m_last_error(self.h) or b"").decode()

    def close(self):
        self.lib.b2m_ctx_destroy(self.h)

    def run(self, c: X.Case):
        """The row's routing and expert launches; -> (K3 lines, K4 lines) of the routed experts, as key/value dicts."""
        es = 4 if c.dtype == "f32" else 2
        x = np.zeros(c.T * c.H * es, dtype=np.uint8)
        out = np.zeros_like(x)
        _take_log(self.lib)
        if c.routed_by_forward:
            lg = X.router_logits(c.counts, c.T, c.k)
            if c.etype == X.DEEPSEEK:
                lg = torch.softmax(lg, dim=-1)
            lg = np.ascontiguousarray(lg.numpy(), dtype=np.float32)
            kind = 2 if c.etype == X.DEEPSEEK else 1
            rc = self.lib.b2m_moe_forward(self.h, 0, x.ctypes.data, lg.ctypes.data, kind, L.DTYPE_F32, c.T, 0, out.ctypes.data, None)
        else:
            m = np.ascontiguousarray(X.route_mask(c.counts, c.T, c.k).numpy().astype(np.uint8))
            rc = self.lib.b2m_route_from_mask(self.h, 0, x.ctypes.data, m.ctypes.data, c.T, None)
            assert rc == 0, self.err()
            rc = self.lib.b2m_run_experts_ex(self.h, 0, c.T, 3, None)
        assert rc == 0, (c.name, self.err())
        gemms = [_kv(ln) for ln in _take_log(self.lib) if ln.startswith("gemm")]
        routed = [g for g in gemms if g["single_n"] == "-1"]
        return [g for g in routed if g["epi"] == "0"], [g for g in routed if g["epi"] == "1"], gemms


def tile_span(dn: dict, sms: int = X.SMS):
    """(units, largest number of CTAs one K4 tile spans) under gemm_body's stream-K partition."""
    nt, M, K = int(dn["nt"]), int(dn["M"]), int(dn["K"])
    step = 256 if dn["dual_m"] == "1" else 128
    m_tiles, kb = -(-M // step), -(-K // 64)
    offs, slots = eval(dn["offsets"]), eval(dn["slot_of"])
    tiles = sum(m_tiles * -(-(offs[e + 1] - offs[e]) // nt) for e in range(len(slots))
                if offs[e + 1] > offs[e] and slots[e] >= 0)
    units = tiles * kb
    span = max(X.stream_k_spans(kb, tiles)) if tiles else 0
    return units, span


def observed_plan(up: dict, dn: dict) -> X.Plan:
    ks, sk = int(dn["ksplit"]), dn["stream_k"] == "1"
    return X.Plan(int(up["nt"]), int(dn["nt"]), ks > 1, sk, dn["dual_m"] == "1", up["early_a"] == "1",
                  dn["early_a"] == "1", tile_span(dn)[1] if sk else 0)


def test_every_row_runs_the_plan_it_claims(sim):
    groups = defaultdict(list)
    for c in X.CASES:
        groups[c.engine_key].append(c)
    bad = []
    for rows in groups.values():
        eng = SimEngine(sim, rows[0], max(c.T for c in rows))
        try:
            for c in rows:
                ups, dns, gemms = eng.run(c)
                assert ups and len(ups) == len(dns), (c.name, gemms)
                # every wave's launches carry the same plan
                plans = {observed_plan(u, d) for u, d in zip(ups, dns)}
                got = plans.pop() if len(plans) == 1 else plans
                units = tile_span(dns[0])[0] if int(dns[0]["nt"]) else 0
                print(f"{c.name:24s} T={c.T:<5d} counts={list(c.counts)[:8]}{'...' if c.E > 8 else ''} launches={len(ups)} "
                      f"units={units} plan={got}")
                assert eval(ups[0]["offsets"]) == [sum(c.counts[:e]) for e in range(c.E + 1)], c.name
                if c.slots:
                    assert len(ups) >= -(-sum(n > 0 for n in c.counts) // c.slots), c.name
                if c.shared:
                    assert sum(g["single_n"] == str(c.T) for g in gemms) == 2, c.name
                if got != c.plan:
                    bad.append((c.name, c.plan, got))
        finally:
            eng.close()
    assert not bad, "rows whose plan differs from the claim:\n" + "\n".join(f"{n}: claims {a}\n{' ' * len(n)}  runs   {b}"
                                                                              for n, a, b in bad)


# ------------------------------------------------------------------------------------------------ coverage
def _tc(c):
    return c.dtype != "f32" and c.gemm_impl == 0


def coverage():
    """item -> the rows covering it"""
    rows = X.CASES
    cov = defaultdict(list)
    for c in rows:
        p = c.plan
        if _tc(c):
            cov[f"K3 tile {p.nt_up}"].append(c.name)
            cov[f"K4 tile {p.nt_dn}"].append(c.name)
            if not p.splitk:
                cov["K4 whole-K"].append(c.name)
            if p.stream_k and not c.slots:      # (offload rows: each wave has its own partition)
                cov["K4 stream-K"].append(c.name)
                kb = -(-c.I // 64)
                tiles = sum(-(-c.H // (256 if p.dual_m else 128)) * -(-n // p.nt_dn) for n in c.counts if n)
                spans = X.stream_k_spans(kb, tiles)
                assert max(spans) == p.span, c.name
                for n, what in ((1, "1 CTA"), (2, "2 CTAs")):
                    if n in spans:
                        cov[f"stream-K tile spans {what}"].append(c.name)
                if max(spans) >= 3:
                    cov["stream-K tile spans >= 3 CTAs"].append(c.name)
                if 15 <= p.span <= 25:
                    cov["stream-K tile spans about 20 CTAs"].append(c.name)
                if tiles * kb < X.SMS:
                    cov["stream-K with fewer units than CTAs"].append(c.name)
            if p.dual_m:
                mt = -(-c.H // 128)
                if c.H % 128:
                    cov["dual_m partial A0, A1 out of range"].append(c.name)
                elif mt % 2:
                    cov["dual_m odd pair count"].append(c.name)
                elif p.stream_k and c.H == X.MH:
                    cov["dual_m even pairs with stream-K at Mixtral H"].append(c.name)
            if p.early_up and p.early_dn and c.T <= 64:
                cov["early-A on for both GEMMs at decode"].append(c.name)
            if not p.early_up and not p.early_dn and c.T > 128:
                cov["early-A off at prefill"].append(c.name)
            if c.H % 128 and c.I % 128 and c.H % 64 and c.I % 64:
                cov[f"M and K tails in both GEMMs, {c.dtype}"].append(c.name)
            fmt = c.fmt if c.dtype == "bf16" else f"{c.fmt}-{c.dtype}"
            if (c.H, c.I) == (X.MH, X.MI):
                cov[f"{fmt} at Mixtral size T={c.T}"].append(c.name)
            if c.H == 384 and p.dual_m:
                cov[f"{fmt} at the odd-pair shape"].append(c.name)
        if c.dtype == "f32":
            cov["fp32 CUDA-core path"].append(c.name)
        if c.gemm_impl == 1:
            cov["gemm_impl=1"].append(c.name)
        nt = c.plan.nt_up or X.pick_nt(c.T)
        if any(n % nt for n in c.counts if n):
            cov["ragged token tiles"].append(c.name)
        if 0 in c.counts:
            cov["empty experts"].append(c.name)
        if c.k > 1 and c.T in c.counts:
            cov["an expert taking every token"].append(c.name)
        if nt in c.counts and nt + 1 in c.counts:
            cov["counts NT and NT+1"].append(c.name)
        cov[f"expert type {c.etype}" + (" with shared expert" if c.shared else "")].append(c.name)
        cov[f"numerics {c.numerics}"].append(c.name)
        if c.slots and c.slots < sum(n > 0 for n in c.counts):
            cov[f"offload waves, {c.slots} slots for {sum(n > 0 for n in c.counts)} active experts"].append(c.name)
    return cov


REQUIRED = (
    [f"K3 tile {n}" for n in (16, 32, 64, 128)] + [f"K4 tile {n}" for n in (16, 32, 64, 128, 256)] +
    ["K4 whole-K", "K4 stream-K", "stream-K tile spans 1 CTA", "stream-K tile spans 2 CTAs", "stream-K tile spans >= 3 CTAs",
     "stream-K tile spans about 20 CTAs", "stream-K with fewer units than CTAs",
     "dual_m even pairs with stream-K at Mixtral H", "dual_m odd pair count", "dual_m partial A0, A1 out of range",
     "early-A on for both GEMMs at decode", "early-A off at prefill",
     "M and K tails in both GEMMs, bf16", "M and K tails in both GEMMs, f16", "ragged token tiles", "empty experts",
     "an expert taking every token", "counts NT and NT+1"] +
    [f"{f} at Mixtral size T={T}" for f in ("bf16", "pk12", "fp8", "int4", "int4-f16") for T in (1, 24, 300, 1100)] +
    [f"{f} at the odd-pair shape" for f in ("bf16", "pk12", "fp8", "int4", "int4-f16")] +
    ["fp32 CUDA-core path", "gemm_impl=1"] +
    ["expert type mixtral", "expert type deepseek with shared expert", "expert type switch", "expert type switch_gated",
     "expert type nllb", "numerics reference", "numerics fp32", "offload waves, 2 slots for 8 active experts"])


def test_rows_cover_every_plan_and_format():
    cov = coverage()
    for item in REQUIRED:
        print(f"{item:48s} {', '.join(cov.get(item, [])) or '-- MISSING'}")
    missing = [item for item in REQUIRED if not cov.get(item)]
    assert not missing, f"coverage items no row reaches: {missing}"


def test_counts_and_router_logits_are_the_designed_ones():
    for c in X.CASES:
        assert len(c.counts) == c.E and sum(c.counts) == c.T * c.k and max(c.counts) <= c.T, c.name
        lg = X.router_logits(c.counts, c.T, c.k)
        top = torch.sort(lg, dim=-1, descending=True).values
        assert bool((top[:, c.k - 1] > top[:, c.k] if c.E > c.k else True).all()), c.name      # no ties at the k-th choice
        idx = torch.topk(lg, c.k, dim=-1).indices
        assert torch.equal(torch.bincount(idx.flatten(), minlength=c.E), torch.tensor(c.counts)), c.name
        assert torch.equal(X.route_mask(c.counts, c.T, c.k).sum(0), torch.tensor(c.counts)), c.name


# ------------------------------------------------------------------------------------------------ reference
def _small(etype, dtype, fmt, numerics="reference"):
    return X.Case(f"small_{etype}_{dtype}_{fmt}", etype, 256, 384, 2, 1, dtype, fmt, 9, (9, 0),
                  X.Plan(0, 0, False, False, False, False, False), numerics=numerics)


SMALL = ([(et, dt, "bf16") for et in X.ETYPE for dt in ("bf16", "f16", "f32")] +
         [(X.MIXTRAL, "bf16", "fp8"), (X.DEEPSEEK, "bf16", "fp8"), (X.MIXTRAL, "bf16", "int4"), (X.MIXTRAL, "f16", "int4"),
          (X.DEEPSEEK, "f16", "int4")])


@pytest.mark.parametrize("etype,dtype,fmt", SMALL)
def test_reference_is_the_oracle_bit_for_bit(etype, dtype, fmt):
    torch.set_num_threads(1)
    c = _small(etype, dtype, fmt)
    ex = X.make_expert(c, seed=7)
    x = X.make_x(c.T, c.H, X.DTYPES[dtype], seed=8)
    hmid, y = X.reference(c, x, ex.w)
    want = O.expert_ffn(x, ex.w, X.ETYPE[etype])
    assert want.dtype == X.DTYPES[dtype]
    assert torch.equal(y.to(want.dtype), want), f"max |diff| {(y - want.float()).abs().max()}"
    # the intermediate and the output are not trivially small: every row saw real sums
    assert bool((hmid.double().abs().amax(dim=1) >= 32).all()) and bool((y.abs().amax(dim=1) > 0).all())
    # the dense down-projection check: the reference of the down GEMM alone is the oracle's matmul too
    h2 = X.make_hmid(c.T, c.I, X.DTYPES[dtype], seed=9)
    _, y2 = X.reference(c, x, ex.w, hmid=h2)
    down = dict(zip([r for r, _ in X.matrix_shapes(etype, c.H, c.I)], ex.w))
    want2 = torch.matmul(h2, down["down"].transpose(0, 1))
    if etype == X.NLLB:
        want2 = want2 + down["bias2"]
    assert torch.equal(y2.to(want2.dtype), want2)


def test_quantised_experts_dequantise_to_the_reference_weights():
    """The fp8 / int4 tensors handed to the engine dequantise (fp8.py / int4.py, the engine's own definitions) to the
    weights the reference computes with."""
    from moe_infinity_b200 import fp8 as F8
    from moe_infinity_b200 import int4 as I4
    for dtype, fmt in (("bf16", "fp8"), ("bf16", "int4"), ("f16", "int4")):
        c = _small(X.MIXTRAL, dtype, fmt)
        ex = X.make_expert(c, seed=11)
        for i, w in enumerate(ex.w):
            if fmt == "fp8":
                got = F8.dequantize_block128(ex.load[i], ex.scales[i], X.DTYPES[dtype])
            else:
                got = I4.dequantize_g128(ex.load[i], ex.scales[i], ex.zeros[i], X.DTYPES[dtype])
            assert torch.equal(got, w), (fmt, dtype, i)
        # the scales really vary inside a matrix
        assert all(len(torch.unique(s.float())) > 1 for s in ex.scales)


def test_reference_refuses_data_outside_the_exact_range():
    c = _small(X.MIXTRAL, "bf16", "bf16")
    ex = X.make_expert(c, seed=3)
    x = X.make_x(c.T, c.H, torch.bfloat16, seed=4)
    with pytest.raises(AssertionError):
        X.reference(c, x * 0, ex.w)                        # g = 0 < 32: SiLU(g) != g
    with pytest.raises(AssertionError):
        X.reference(c, x * 64, ex.w)                       # g up to 64 * 216: not exact in bf16 / over the budget
