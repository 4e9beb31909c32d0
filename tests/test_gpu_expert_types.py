"""GPU parity of every expert type of the boundary (expert_module.h:13-18) against the reference's OWN modules.

Expected outputs come from tests/golden/expert_ffn_ref.pt = /root/reference/core/parallel/expert_module.cpp compiled as-is
and run on CPU (tests/golden/make_expert_golden.py); a second, differently seeded expert is checked against the oracle
(which tests/test_oracle_expert_ref.py pins bit-for-bit to the same compiled reference).  Path under test: the staged
C-ABI calls the reference's dispatcher maps to -- b2m_route_from_mask -> b2m_run_experts -> b2m_expert_outputs
(expert_executor.py:46-56).  Tolerance: the hidden-state bound of tests/test_gpu_parity.py (2 ulp bf16 / 1e-3 fp16).
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import expert_cases as C  # noqa: E402
from oracle import moe_oracle as O  # noqa: E402
from test_gpu_parity import hidden_close  # noqa: E402

GOLD = torch.load(os.path.join(HERE, "golden", "expert_ffn_ref.pt"))
HALF_CASES = sorted(n for n, c in C.CASES.items() if c[1] != 1)      # the tensor-core path runs bf16 / f16 experts
F32_CASES = sorted(n for n, c in C.CASES.items() if c[1] == 1)        # dtype int 1: CUDA-core fp32 path (f32_path.cu)


def f32_close(y, y_ref, what=""):
    """fp32 experts: both sides are fp32 FMA chains over K <= a few thousand terms in different orders."""
    y, y_ref = y.float().cpu().reshape(-1), y_ref.float().reshape(-1)
    rms = y_ref.pow(2).mean().sqrt().item()
    diff = (y - y_ref).abs()
    bound = 2e-5 * y_ref.abs() + 2e-5 * rms
    assert bool((diff <= bound).all()), f"{what}: max diff {diff.max().item():.3e} (rms {rms:.3e})"


def _second_expert(ws, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(w.shape, generator=g) * (0.3 if w.dim() == 1 else 0.08)).to(w.dtype) for w in ws]


# id "tcgen05" = gemm_impl 0, the tensor-core product path (wgmma on sm_90a); the name is kept so the test
# ids stay the same across GPU architectures
@pytest.mark.parametrize("impl", [0, 1], ids=["tcgen05", "simt"])
@pytest.mark.parametrize("name", HALF_CASES)
def test_expert_type_outputs_match_reference_module(lib_built, name, impl):
    from moe_infinity_b200 import MoEEngine
    et, di, ws, x = C.make_case(name)
    dt = C.DT[di]
    n, H = x.shape
    I = ws[0].shape[0]
    ws2 = _second_expert(ws, 900 + C.CASES[name][5])
    eng = MoEEngine(num_layers=1, num_experts=2, hidden=H, inter=I, top_k=2, dtype=dt, expert_type=et,
                    max_tokens=max(n, 16), gemm_impl=impl)
    eng.load_expert(0, 0, ws)
    eng.load_expert(0, 1, ws2)
    mask = torch.zeros(n, 2, dtype=torch.bool)
    mask[:, 0] = True                      # expert 0 sees every row  -> compare with the golden reference output
    mask[::2, 1] = True                    # expert 1 sees rows 0,2,4,... (ascending token order)
    eng.route_from_mask(0, x.cuda(), mask.cuda())
    eng.run_experts(0, n)
    rows, offs = eng.expert_outputs(n)
    torch.cuda.synchronize()
    assert offs == [0, n, n + (n + 1) // 2]
    hidden_close(rows[offs[0]:offs[1]], GOLD[name]["y"], None, dt, f"{name} expert 0 vs compiled reference")
    want1 = O.expert_ffn(x[::2], ws2, et)
    hidden_close(rows[offs[1]:offs[2]], want1, None, dt, f"{name} expert 1 vs oracle")


@pytest.mark.parametrize("et", [2, 3])
def test_bias_experts_fused_forward(lib_built, et):
    """NLLB / FSGPT experts through the fused call with a Mixtral-style router (softmax, top-2, renormalise)."""
    from moe_infinity_b200 import MoEEngine, _lib as L
    torch.manual_seed(5 + et)
    dt, E, k, H, I, T = torch.bfloat16, 4, 2, 128, 192, 40
    g = torch.Generator().manual_seed(40 + et)
    experts = [[(torch.randn(I, H, generator=g) * 0.06).to(dt), (torch.randn(I, generator=g) * 0.2).to(dt),
                (torch.randn(H, I, generator=g) * 0.06).to(dt), (torch.randn(H, generator=g) * 0.2).to(dt)]
               for _ in range(E)]
    x = torch.randn(1, T, H, generator=g).to(dt)
    logits = torch.randn(T, E, generator=g).to(dt)
    r = O.mixtral_route(logits, k, dt)
    # reference combine: final[idx] += out_e * w  (mixtral.py:96-101), ascending expert id
    final = torch.zeros(T, H, dtype=dt)
    for out_e, _, e, _ in O.dispatch_local(x.reshape(T, H), r.router_mask, experts, et):
        idx = r.router_mask[:, e].bool()
        final[idx] += out_e * r.routing_weights_mask[idx, e][:, None]
    eng = MoEEngine(num_layers=1, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dt, expert_type=et,
                    router=L.ROUTER_MIXTRAL, max_tokens=64)
    for e in range(E):
        eng.load_expert(0, e, experts[e])
    out = eng.forward(0, x.cuda(), router_logits=logits.cuda())
    torch.cuda.synchronize()
    tied = O.tied_tokens(r.scores, k)
    hidden_close(out.reshape(T, H)[(~tied).cuda()], final[~tied], None, dt, f"bias expert type {et} fused forward")


@pytest.mark.parametrize("name", F32_CASES)
def test_fp32_expert_type_outputs_match_reference_module(lib_built, name):
    """dtype int 1 (Switch-base-8's default dtype, expert_module.h:21): all six expert types in fp32 through the same
    staged C-ABI calls, against the reference's compiled modules (expert 0) and the oracle (expert 1)."""
    from moe_infinity_b200 import MoEEngine
    et, di, ws, x = C.make_case(name)
    assert C.DT[di] == torch.float32
    n, H = x.shape
    I = ws[0].shape[0]
    ws2 = _second_expert(ws, 900 + C.CASES[name][5])
    eng = MoEEngine(num_layers=1, num_experts=2, hidden=H, inter=I, top_k=2, dtype=torch.float32, expert_type=et,
                    max_tokens=max(n, 16))
    eng.load_expert(0, 0, ws)
    eng.load_expert(0, 1, ws2)
    mask = torch.zeros(n, 2, dtype=torch.bool)
    mask[:, 0] = True
    mask[::2, 1] = True
    eng.route_from_mask(0, x.cuda(), mask.cuda())
    eng.run_experts(0, n)
    rows, offs = eng.expert_outputs(n)
    torch.cuda.synchronize()
    assert offs == [0, n, n + (n + 1) // 2] and rows.dtype == torch.float32
    f32_close(rows[offs[0]:offs[1]], GOLD[name]["y"], f"{name} expert 0 vs compiled reference")
    f32_close(rows[offs[1]:offs[2]], O.expert_ffn(x[::2], ws2, et), f"{name} expert 1 vs oracle")


def test_config1_switch_base8_fp32_through_the_plugin(lib_built):
    """BASELINE config 1 on the GPU: Switch-base-8 shapes (d_model 768, d_ff 3072, 8 experts, capacity 64), one sparse
    layer, seq 128 batch 1, fp32 -- fused forward vs the oracle block (pinned to the literal reference block by
    tests/test_oracle_golden.py::test_literal_switch_block_equals_oracle)."""
    from moe_infinity_b200 import MoEEngine, _lib as L
    D, Fd, E, cap, B, S = 768, 3072, 8, 64, 1, 128
    experts = O.make_experts(E, D, Fd, torch.float32, 77, O.SWITCH_DENSE_ACT_DENSE, std=0.05)
    g = torch.Generator().manual_seed(78)
    hidden = torch.randn(B, S, D, generator=g)
    gate = torch.randn(E, D, generator=g) * 0.1
    want, (logits, expert_index), mask = O.switch_block(hidden, gate, experts, cap)
    eng = MoEEngine(num_layers=1, num_experts=E, hidden=D, inter=Fd, top_k=1, dtype=torch.float32,
                    expert_type=L.EXPERT_SWITCH, router=L.ROUTER_SWITCH_TOP1, expert_capacity=cap, max_tokens=B * S)
    for e in range(E):
        eng.load_expert(0, e, experts[e])
    out = eng.forward(0, hidden.cuda(), router_logits=logits.reshape(-1, E).cuda(), seq_len=S)
    torch.cuda.synchronize()
    idx = eng.ws("topk_idx", B * S).cpu().flatten()
    kept = mask.reshape(-1, E).any(-1)
    assert torch.equal(idx[kept].long(), expert_index.flatten()[kept]), "expert index assignment differs"
    assert bool((idx[~kept] < 0).all()), "tokens beyond the expert capacity must be dropped"
    f32_close(out, want, "config 1 (Switch-base-8 fp32)")
