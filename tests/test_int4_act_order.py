"""CPU: act-order GPTQ (desc_act=True) experts on the f16 int4 format (B2M_WEIGHTS_INT4_G128_F16).

* int4.from_gptq_act_order against a test-side act-order packer (tests/act_order_packers.py), v1 and v2: the columns of
  W[:, perm] have contiguous 128-column groups, and undoing the permutation gives GPTQ's own fp16 dequantisation bit for
  bit; int4.dequantize_g_idx gives it directly; the refusals;
* hf.load_int4_checkpoint(act_order=True) on synthetic Mixtral and DeepSeek shards, checked against a recording engine:
  the stored matrices are w1[P2][:, P], w3[P2][:, P] and w2[:, P2], the gather tables are P per expert and only layers
  with a non-identity P get one, shared experts are dequantised in natural order, and experts whose gate and up
  projections have different g_idx are refused; with act_order=False the refusal names act_order=True;
* MoEEngine.set_input_perm refuses tables that are not row-wise permutations of 0..H-1."""
from __future__ import annotations

import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import act_order_packers as A  # noqa: E402
import int4_checkpoint_packers as P  # noqa: E402
from moe_infinity_b200 import _lib as L  # noqa: E402
from moe_infinity_b200 import hf  # noqa: E402
from moe_infinity_b200.engine import MoEEngine  # noqa: E402
from moe_infinity_b200.int4 import (_pack_codes, dequantize_g128, dequantize_g_idx, from_gptq,  # noqa: E402
                                    from_gptq_act_order)

GPTQ_CFG = dict(quant_method="gptq", bits=4, group_size=128, desc_act=True, sym=False, checkpoint_format="gptq")


def _bits(w: torch.Tensor) -> torch.Tensor:
    return w.view(torch.int16)


def _perm_of(g_idx: torch.Tensor) -> torch.Tensor:
    return torch.sort(g_idx.long(), stable=True).indices


@pytest.mark.parametrize("fmt", ["gptq", "gptq_v2"])
def test_from_gptq_act_order_roundtrip(fmt):
    g = torch.Generator().manual_seed(["gptq", "gptq_v2"].index(fmt) + 40)
    out, n_in = 256, 640
    order, g_idx = A.random_g_idx(n_in, g)
    q, s, z = P.random_qsz(out, n_in, g, z_lo=1 if fmt == "gptq" else 0)
    s[0, 0] = -s[0, 0].abs() - 0.01                        # a negative scale, a subnormal one, large ones
    s[1, 1] = torch.tensor(3e-7, dtype=torch.float16)
    s[2, :] = torch.tensor(4000.0, dtype=torch.float16)
    ck = A.gptq_act_order_pack(q, s, z, g_idx, v1=fmt == "gptq")
    q2, s2, z2, perm = from_gptq_act_order(*ck, checkpoint_format=fmt)
    assert perm.dtype == torch.int64 and torch.equal(perm, _perm_of(g_idx))
    assert torch.equal(g_idx.long()[perm], torch.arange(n_in) // 128)     # W[:, perm] has contiguous groups
    assert q2.shape == (out, n_in // 2) and torch.equal(_bits(s2), _bits(s)) and torch.equal(z2.long(), z)
    want = A.fp16_dequant_g_idx(q, s, z, g_idx)
    got = dequantize_g128(q2, s2, z2, torch.float16)
    assert torch.equal(_bits(got), _bits(want[:, perm]))
    assert torch.equal(_bits(got[:, perm.argsort()]), _bits(want))
    assert torch.equal(_bits(dequantize_g_idx(_pack_codes(q), s2, z2, g_idx)), _bits(want))
    # a natural-order g_idx is an identity permutation, and from_gptq still refuses act-order
    nat = (torch.arange(n_in) // 128).to(torch.int32)
    assert torch.equal(from_gptq_act_order(*ck[:3], nat, checkpoint_format=fmt)[3], torch.arange(n_in))
    with pytest.raises(ValueError, match="act-order"):
        from_gptq(*ck, checkpoint_format=fmt)


def test_from_gptq_act_order_refusals():
    g = torch.Generator().manual_seed(41)
    _, g_idx = A.random_g_idx(256, g)
    q, s, z = P.random_qsz(128, 256, g, z_lo=1)
    qw, qz, sc, gi = A.gptq_act_order_pack(q, s, z, g_idx)
    uneven = gi.clone()
    uneven[(gi == 1).nonzero()[0]] = 0                      # 129 columns in group 0, 127 in group 1
    with pytest.raises(ValueError, match="exactly 128"):
        from_gptq_act_order(qw, qz, sc, uneven)
    out_of_range = gi.clone()
    out_of_range[0] = 2
    with pytest.raises(ValueError, match="exactly 128"):
        from_gptq_act_order(qw, qz, sc, out_of_range)
    with pytest.raises(ValueError, match="g_idx"):
        from_gptq_act_order(qw, qz, sc, gi[:128])
    with pytest.raises(ValueError, match="g_idx"):
        from_gptq_act_order(qw, qz, sc, gi.float())
    with pytest.raises(ValueError, match="int32"):
        from_gptq_act_order(qw.to(torch.int64), qz, sc, gi)
    with pytest.raises(ValueError, match="group size"):
        from_gptq_act_order(qw, qz, torch.cat([sc, sc]), gi)
    with pytest.raises(ValueError, match="g_idx"):
        dequantize_g_idx(_pack_codes(q), s, z.to(torch.uint8), gi[:128])


# ---------------------------------------------------------------- hf.load_int4_checkpoint(act_order=True)
class _FakeEngine:
    """Records what load_int4_checkpoint hands an engine (the real one needs a GPU)."""

    def __init__(self, L_, E, H, I, expert_type, shared_inter=0, router=L.ROUTER_MIXTRAL):
        self.int4, self.dtype = True, torch.float16
        self.L, self.E, self.H, self.I = L_, E, H, I
        self.expert_type, self.shared_inter, self.router = expert_type, shared_inter, router
        self.experts, self.shared, self.gates, self.perms, self.resident = {}, {}, {}, {}, {}

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

    def set_input_perm(self, l, perm):
        self.perms[l] = perm

    def stored(self, l, e):
        """The three matrices the engine holds for expert (l, e), dequantised as it computes with them."""
        return [dequantize_g128(q, s, z, torch.float16) for q, s, z in zip(*self.experts[(l, e)])]


def _mixtral_act_order(L_=2, E=3, H=256, I=384, seed=50, mismatch=None):
    """Layer 0: every expert act-order in gate/up (P) and down (P2).  Layer 1: gate/up in natural order (no table),
    down act-order.  `mismatch` = (layer, expert) whose w3 gets a g_idx of its own."""
    g = torch.Generator().manual_seed(seed)
    tensors, truth, perms = {}, {}, {}
    nat_h = (torch.arange(H) // 128).to(torch.int32)
    for l in range(L_):
        base = f"model.layers.{l}.block_sparse_moe"
        tensors[f"{base}.gate.weight"] = torch.randn(E, H, generator=g).to(torch.float16)
        for e in range(E):
            gi = A.random_g_idx(H, g)[1] if l == 0 else nat_h
            gi2 = A.random_g_idx(I, g)[1]
            gi3 = A.random_g_idx(H, g)[1] if mismatch == (l, e) else gi
            perms[(l, e)] = (_perm_of(gi), _perm_of(gi2))
            pre = f"{base}.experts.{e}"
            A.put_linear(tensors, truth, f"{pre}.w1", I, H, g, gi)
            A.put_linear(tensors, truth, f"{pre}.w2", H, I, g, gi2)
            A.put_linear(tensors, truth, f"{pre}.w3", I, H, g, gi3)
    return tensors, truth, perms


@pytest.mark.parametrize("resident", [True, False])
def test_load_act_order_mixtral(tmp_path, resident):
    H, I = 256, 384
    tensors, truth, perms = _mixtral_act_order(H=H, I=I)
    eng = _FakeEngine(2, 3, H, I, L.EXPERT_MIXTRAL)
    assert hf.load_int4_checkpoint(eng, P.write_shards(str(tmp_path), tensors), GPTQ_CFG, "mixtral", resident=resident,
                                   act_order=True) == [0, 1]
    assert all(v == resident for v in eng.resident.values()) and len(eng.experts) == 6
    for (l, e), (p, p2) in perms.items():
        pre = f"model.layers.{l}.block_sparse_moe.experts.{e}"
        w1, w2, w3 = eng.stored(l, e)
        assert torch.equal(_bits(w1), _bits(truth[f"{pre}.w1"][p2][:, p])), (l, e)
        assert torch.equal(_bits(w3), _bits(truth[f"{pre}.w3"][p2][:, p])), (l, e)
        assert torch.equal(_bits(w2), _bits(truth[f"{pre}.w2"][:, p2])), (l, e)
    assert sorted(eng.perms) == [0]                        # layer 1's gate/up are in natural order: no table
    assert eng.perms[0].shape == (3, H)
    for e in range(3):
        assert torch.equal(eng.perms[0][e].long(), perms[(0, e)][0])


def test_load_act_order_deepseek(tmp_path):
    """DeepSeek layout (gate | up | down), GPTQ v2, a dense first layer, act-order shared experts dequantised in natural
    order."""
    g = torch.Generator().manual_seed(51)
    H, I, Is, E = 256, 128, 256, 4
    tensors, truth, perms = {"model.layers.0.mlp.gate_proj.weight": torch.zeros(4, 4, dtype=torch.float16)}, {}, {}
    base = "model.layers.1.mlp"
    tensors[f"{base}.gate.weight"] = torch.randn(E, H, generator=g)
    for e in range(E):
        gi, gi2 = A.random_g_idx(H, g)[1], A.random_g_idx(I, g)[1]
        perms[e] = (_perm_of(gi), _perm_of(gi2))
        for n, (o, i), gx in (("gate_proj", (I, H), gi), ("up_proj", (I, H), gi), ("down_proj", (H, I), gi2)):
            A.put_linear(tensors, truth, f"{base}.experts.{e}.{n}", o, i, g, gx, v1=False)
    for n, (o, i) in (("gate_proj", (Is, H)), ("up_proj", (Is, H)), ("down_proj", (H, Is))):
        A.put_linear(tensors, truth, f"{base}.shared_experts.{n}", o, i, g, A.random_g_idx(i, g)[1], v1=False)
    eng = _FakeEngine(2, E, H, I, L.EXPERT_DEEPSEEK, shared_inter=Is, router=L.ROUTER_DEEPSEEK_GREEDY)
    cfg = dict(GPTQ_CFG, checkpoint_format="gptq_v2")
    assert hf.load_int4_checkpoint(eng, P.write_shards(str(tmp_path), tensors, nshards=3), cfg, "deepseek_v2",
                                   act_order=True) == [1]
    for e, (p, p2) in perms.items():
        pre = f"{base}.experts.{e}"
        wg, wu, wd = eng.stored(1, e)
        assert torch.equal(_bits(wg), _bits(truth[f"{pre}.gate_proj"][p2][:, p]))
        assert torch.equal(_bits(wu), _bits(truth[f"{pre}.up_proj"][p2][:, p]))
        assert torch.equal(_bits(wd), _bits(truth[f"{pre}.down_proj"][:, p2]))
        assert torch.equal(eng.perms[1][e].long(), p)
    for n, w in zip(("gate_proj", "up_proj", "down_proj"), eng.shared[1]):
        assert w.dtype == torch.float16 and torch.equal(_bits(w), _bits(truth[f"{base}.shared_experts.{n}"]))


def test_load_act_order_refusals(tmp_path):
    tensors, _, _ = _mixtral_act_order(L_=1, E=2, mismatch=(0, 1))
    shards = P.write_shards(str(tmp_path), tensors)
    eng = _FakeEngine(1, 2, 256, 384, L.EXPERT_MIXTRAL)
    with pytest.raises(ValueError, match="layer 0 expert 1: w1 and w3 have different g_idx"):
        hf.load_int4_checkpoint(eng, shards, GPTQ_CFG, "mixtral", act_order=True)
    with pytest.raises(ValueError, match=r"act-order.*act_order=True"):
        hf.load_int4_checkpoint(_FakeEngine(1, 2, 256, 384, L.EXPERT_MIXTRAL), shards, GPTQ_CFG, "mixtral")


def test_set_input_perm_refuses_non_permutations():
    eng = object.__new__(MoEEngine)            # the checks run before the library is called
    eng.E, eng.H = 2, 256
    good = torch.stack([torch.randperm(256), torch.arange(256)])
    dup = good.clone()
    dup[0, 0] = dup[0, 1]
    with pytest.raises(ValueError, match="permutation of 0..H-1"):
        eng.set_input_perm(0, dup)
    big = good.clone()
    big[1, 5] = 256
    with pytest.raises(ValueError, match="permutation of 0..H-1"):
        eng.set_input_perm(0, big)
    with pytest.raises(ValueError, match=r"\[2, 256\]"):
        eng.set_input_perm(0, good[:1])
    with pytest.raises(ValueError, match="integer"):
        eng.set_input_perm(0, good.float())
