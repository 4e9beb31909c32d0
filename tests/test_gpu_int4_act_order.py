"""GPU: act-order GPTQ experts on the f16 int4 format (B2M_WEIGHTS_INT4_G128_F16 with b2m_set_input_perm).

An act-order expert is stored as w1[P2][:, P], w3[P2][:, P] and w2[:, P2] (P: the gate/up input order, P2: the down
projection's), and the routing kernels gather each of its rows as x[t][P].  Checked:
* the gather: after `route` (both routing paths, T from 1 to 1024) and `route_from_mask`, every "xp" row is
  x[perm_token[row]][P_e] exactly, and a layer without a table gathers natural rows;
* exactness: a full-size Mixtral layer (H=4096, I=14336, E=8, k=2) from T=1 to 1024 against an f16 engine holding the
  dequantised permuted matrices whose "xp" rows are overwritten with the permuted rows between route and run_experts:
  gate/up outputs bit for bit, routed expert outputs bit for bit whenever both engines reproduce their own, layer output
  equal or within hidden_close;
* the same layer against an f16 engine holding GPTQ's natural-order weights: only the fp32 summation order differs;
* synthetic act-order GPTQ checkpoints (Mixtral, and DeepSeek-V2-Lite shaped with f16 shared experts) through
  hf.load_int4_checkpoint(act_order=True), offloaded against resident experts, a captured decode session, and an
  out-of-range table entry reported by b2m_check_errors as B2M_EINVAL without a fault."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

H, I, E, K = 4096, 14336, 8, 2
DT = torch.float16


def _engine(int4, H=H, I=I, E=E, K=K, L=1, max_tokens=1024, **kw):
    from moe_infinity_b200 import MoEEngine
    if int4:
        return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                         expert_dtype=torch.uint4, **kw)
    return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                     pack_weights=False, **kw)


def _x(T, Hx=H, seed=0):
    return torch.randn(T, Hx, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1000 * seed + T)).to(DT)


def _perms(n, length, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.stack([torch.randperm(length, generator=g, device="cuda") for _ in range(n)])


def _expected_xp(eng, x, T, table):
    """x[perm_token[row]][P_e] for every routed row (natural rows where table is None)."""
    pt = eng.ws("perm_token", T).long()
    off = eng.ws("offsets", T).tolist()
    want = torch.zeros(off[-1], x.shape[1], dtype=DT, device="cuda")
    for e in range(eng.E):
        rows = slice(off[e], off[e + 1])
        src = x[pt[rows]]
        want[rows] = src if table is None else src[:, table[e]]
    return want, off[-1]


def test_gather_rows(lib_built):
    Hs, Es, Ks = 1024, 8, 2
    eng = _engine(True, H=Hs, I=256, E=Es, K=Ks, L=2)
    table = _perms(Es, Hs, 1)
    eng.set_input_perm(0, table)
    gate = (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT)
    for l in range(2):
        eng.set_gate(l, gate)
    for T in (1, 8, 64, 256, 257, 1024):
        x = _x(T, Hs)
        for l, tb in ((0, table), (1, None)):
            eng.route(l, x)
            torch.cuda.synchronize()
            want, n = _expected_xp(eng, x, T, tb)
            assert n == T * Ks and torch.equal(eng.ws("xp", T)[:n], want), (T, l)
        mask = torch.zeros(T, Es, dtype=torch.uint8, device="cuda")
        mask[torch.arange(T), torch.arange(T) % Es] = 1
        mask[torch.arange(T), (torch.arange(T) * 3 + 1) % Es] = 1
        eng.route_from_mask(0, x, mask)
        torch.cuda.synchronize()
        want, n = _expected_xp(eng, x, T, table)
        assert torch.equal(eng.ws("xp", T)[:n], want), ("mask", T)
    eng.set_input_perm(0, None)
    x = _x(64, Hs)
    eng.route(0, x)
    torch.cuda.synchronize()
    want, n = _expected_xp(eng, x, 64, None)
    assert torch.equal(eng.ws("xp", 64)[:n], want)
    eng.close()


def _act_order_layer(seed, H=H, I=I, E=E, shapes=None):
    """Per expert: stored (q, s, z) of [w1[P2][:, P], w2[:, P2], w3[P2][:, P]] (Mixtral order) and (P, P2)."""
    from moe_infinity_b200.int4 import quantize_g128
    g = torch.Generator(device="cuda").manual_seed(seed)
    P, P2 = _perms(E, H, seed + 1), _perms(E, I, seed + 2)
    shapes = shapes or [(I, H), (H, I), (I, H)]
    ws = []
    for e in range(E):
        qsz = [quantize_g128(torch.randn(*shp, generator=g, device="cuda") * 0.02, scale_dtype=DT) for shp in shapes]
        ws.append(tuple(zip(*qsz)))
    return ws, P, P2


def _deq(ws):
    from moe_infinity_b200.int4 import dequantize_g128
    return [[dequantize_g128(q, s, z, DT) for q, s, z in zip(*ex)] for ex in ws]


def _natural(w, p, p2):
    """Stored Mixtral matrices [w1[P2][:, P], w2[:, P2], w3[P2][:, P]] -> the natural-order model's w1, w2, w3."""
    ip, ip2 = p.argsort(), p2.argsort()
    return [w[0][ip2][:, ip], w[1][:, ip2], w[2][ip2][:, ip]]


def _staged(eng, x, T, layer=0, table=None):
    """route -> (xp rows overwritten with the permuted rows when table is given) -> run_experts -> combine."""
    eng.route(layer, x)
    if table is not None:
        want, n = _expected_xp(eng, x, T, table)
        eng.ws("xp", T)[:n].copy_(want)
    eng.run_experts(layer, T)
    out = eng.combine(layer, x)
    torch.cuda.synchronize()
    return out.clone(), eng.ws("hmid", T).clone(), eng.ws("y", T).clone()


def test_fullsize_mixtral_exact_and_natural(lib_built):
    from test_gpu_parity import hidden_close
    ws, P, P2 = _act_order_layer(3)
    deq = _deq(ws)
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    a, b = _engine(True), _engine(False)
    for e, (qs, ss, zs) in enumerate(ws):
        a.load_expert(0, e, qs, scales=ss, zeros=zs)
        b.load_expert(0, e, deq[e])
    a.set_input_perm(0, P)
    for eng in (a, b):
        eng.set_gate(0, gate)
    worst = 0.0
    for T in (1, 2, 8, 16, 64, 128, 256, 1024):
        x = _x(T)
        oa, ha, ya = _staged(a, x, T)
        _, _, ya2 = _staged(a, x, T)
        ob, hb, yb = _staged(b, x, T, table=P)
        _, _, yb2 = _staged(b, x, T, table=P)
        assert torch.isfinite(oa.float()).all() and oa.float().abs().max() > 0, T
        assert torch.equal(ha, hb), f"T={T}: gate/up outputs differ"
        if torch.equal(ya, ya2) and torch.equal(yb, yb2):
            assert torch.equal(ya, yb), f"T={T}: routed expert outputs differ"
        if not torch.equal(oa, ob):
            hidden_close(oa, ob.cpu(), None, DT, f"T={T}")
        fa = a.forward(0, x)
        torch.cuda.synchronize()
        if not torch.equal(fa, oa):
            hidden_close(fa, oa.cpu(), None, DT, f"T={T} forward")
    b.close()
    # the natural-order model: same weights, same routing, different fp32 summation order in the GEMMs
    c = _engine(False)
    for e in range(E):
        c.load_expert(0, e, _natural(deq[e], P[e], P2[e]))
    c.set_gate(0, gate)
    outs = []
    for T in (1, 8, 64, 1024):
        x = _x(T, seed=1)
        oa, oc = a.forward(0, x).clone(), c.forward(0, x).clone()
        torch.cuda.synchronize()
        assert torch.equal(a.ws("topk_idx", T), c.ws("topk_idx", T))
        outs.append((oa, oc))
        worst = max(worst, (oa.float() - oc.float()).abs().max().item())
    # one hidden_close over the whole sweep: a flipped f16 rounding of an intermediate is a few-ulp outlier, and the bound
    # counts such outliers per 10^4 elements (T=1 alone has 4096)
    hidden_close(torch.cat([o for o, _ in outs]), torch.cat([o for _, o in outs]).cpu(), None, DT, "natural-order model")
    print(f"act-order vs natural-order f16 model: largest |difference| {worst:.3e}")
    a.close(); c.close()


def _mixtral_checkpoint(tmp_path, Lc=2, Ec=8, Hc=1024, Ic=2048):
    import act_order_packers as A
    import int4_checkpoint_packers as P
    g = torch.Generator().manual_seed(12)
    tensors, truth = {}, {}
    for l in range(Lc):
        base = f"model.layers.{l}.block_sparse_moe"
        tensors[f"{base}.gate.weight"] = (torch.randn(Ec, Hc, generator=g) * 0.05).to(DT)
        for e in range(Ec):
            gi, gi2 = A.random_g_idx(Hc, g)[1], A.random_g_idx(Ic, g)[1]
            pre = f"{base}.experts.{e}"
            A.put_linear(tensors, truth, f"{pre}.w1", Ic, Hc, g, gi, s_std=0.0015)
            A.put_linear(tensors, truth, f"{pre}.w2", Hc, Ic, g, gi2, s_std=0.0015)
            A.put_linear(tensors, truth, f"{pre}.w3", Ic, Hc, g, gi, s_std=0.0015)
    return P.write_shards(str(tmp_path), tensors), tensors, truth


CFG = dict(quant_method="gptq", bits=4, group_size=128, desc_act=True, checkpoint_format="gptq")


def test_checkpoint_mixtral_resident_offload_graph(tmp_path, lib_built):
    from moe_infinity_b200 import DecodeSession
    from moe_infinity_b200.hf import load_int4_checkpoint
    from test_gpu_parity import hidden_close
    Lc, Ec, Hc, Ic = 2, 8, 1024, 2048
    shards, tensors, truth = _mixtral_checkpoint(tmp_path, Lc, Ec, Hc, Ic)
    kw = dict(H=Hc, I=Ic, E=Ec, K=2, L=Lc, max_tokens=64)
    a, off, nat = _engine(True, **kw), _engine(True, num_slots=3, **kw), _engine(False, **kw)
    assert load_int4_checkpoint(a, shards, CFG, "mixtral", act_order=True) == [0, 1]
    assert load_int4_checkpoint(off, shards, CFG, "mixtral", resident=False, act_order=True) == [0, 1]
    assert sorted(a._perms) == [0, 1]
    for l in range(Lc):
        base = f"model.layers.{l}.block_sparse_moe"
        for e in range(Ec):
            nat.load_expert(l, e, [truth[f"{base}.experts.{e}.{n}"].cuda() for n in ("w1", "w2", "w3")])
        nat.set_gate(l, tensors[f"{base}.gate.weight"])
    for step in range(2):
        for l in range(Lc):
            for T in (8, 64):
                x = _x(T, Hc, seed=10 * step + l)
                oa, oo, on = a.forward(l, x).clone(), off.forward(l, x).clone(), nat.forward(l, x).clone()
                torch.cuda.synchronize()
                if not torch.equal(oa, oo):
                    hidden_close(oo, oa.cpu(), None, DT, f"offload layer {l} T={T}")
                hidden_close(oa, on.cpu(), None, DT, f"checkpoint vs natural layer {l} T={T}")
    st = off.stats()
    assert st["misses"] > 3 and st["evictions"] > 0
    off.close(); nat.close()
    # A captured decode step against eager calls.  The gate/up GEMM is deterministic, so the last layer's gate/up output
    # (computed from rows gathered through its table) must match bit for bit; the layer outputs go through the down
    # projection's split-K fp32 atomics, whose order (and so the last bit of a few elements) varies from run to run even
    # between two eager calls, so they are equal or within hidden_close.
    sess = DecodeSession(a, 8)
    sess.x_host.copy_(torch.randn(Lc, 8, Hc).to(DT))
    eager = torch.stack([a.forward(l, sess.x_host[l].cuda()).clone() for l in range(Lc)]).cpu()
    h_eager = a.ws("hmid", 8).clone()
    sess.capture()
    for _ in range(2):
        out = sess.step().clone()
        assert torch.equal(a.ws("hmid", 8), h_eager)
        if not torch.equal(out, eager):
            hidden_close(out, eager, None, DT, "graph replay")
    a.close()


def test_checkpoint_deepseek_lite(tmp_path, lib_built):
    """DeepSeek-V2-Lite shapes: E=64, k=6, H=2048, I=1408, act-order shared experts (I=2816) dequantised to f16."""
    import act_order_packers as A
    import int4_checkpoint_packers as P
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200.hf import load_int4_checkpoint
    from test_gpu_parity import hidden_close
    Hd, Id, Ed, Kd, Is = 2048, 1408, 64, 6, 2816
    g = torch.Generator().manual_seed(13)
    tensors, truth = {"model.layers.0.mlp.gate_proj.weight": torch.zeros(8, 8, dtype=DT)}, {}
    base = "model.layers.1.mlp"
    tensors[f"{base}.gate.weight"] = torch.randn(Ed, Hd, generator=g) * 0.05
    names = ("gate_proj", "up_proj", "down_proj")
    for e in range(Ed):
        gi, gi2 = A.random_g_idx(Hd, g)[1], A.random_g_idx(Id, g)[1]
        for n, (o, i), gx in zip(names, ((Id, Hd), (Id, Hd), (Hd, Id)), (gi, gi, gi2)):
            A.put_linear(tensors, truth, f"{base}.experts.{e}.{n}", o, i, g, gx, v1=False, s_std=0.0015)
    for n, (o, i) in zip(names, ((Is, Hd), (Is, Hd), (Hd, Is))):
        A.put_linear(tensors, truth, f"{base}.shared_experts.{n}", o, i, g, A.random_g_idx(i, g)[1], v1=False, s_std=0.0015)
    shards = P.write_shards(str(tmp_path), tensors, nshards=3)
    kw = dict(H=Hd, I=Id, E=Ed, K=Kd, L=2, max_tokens=512, expert_type=L.EXPERT_DEEPSEEK,
              router=L.ROUTER_DEEPSEEK_GROUP, n_group=8, topk_group=3, shared_inter=Is)
    a, nat = _engine(True, **kw), _engine(False, **kw)
    cfg = dict(CFG, checkpoint_format="gptq_v2")
    assert load_int4_checkpoint(a, shards, cfg, "deepseek_v2", act_order=True) == [1]
    for e in range(Ed):
        nat.load_expert(1, e, [truth[f"{base}.experts.{e}.{n}"].cuda() for n in names])
    nat.register_shared(1, [truth[f"{base}.shared_experts.{n}"] for n in names])
    nat.set_gate(1, tensors[f"{base}.gate.weight"])
    for T in (1, 8, 512):
        x = _x(T, Hd, seed=2)
        oa, on = a.forward(1, x).clone(), nat.forward(1, x).clone()
        torch.cuda.synchronize()
        hidden_close(oa, on.cpu(), None, DT, f"deepseek T={T}")
    a.close(); nat.close()


def test_out_of_range_entry_is_reported(lib_built):
    from moe_infinity_b200 import _lib as L
    Hs, Es = 1024, 8
    eng = _engine(True, H=Hs, I=256, E=Es, K=2, max_tokens=64)
    eng.set_gate(0, (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT))
    table = torch.arange(Hs, dtype=torch.int32).repeat(Es, 1)
    table[:, 7] = Hs + 5                           # past the row: would read the next token's (or the guard's) elements
    dev = table.to(torch.uint16).cuda()
    big = torch.randn(9, Hs, device="cuda").to(DT)  # x is rows 0..7 of a larger tensor the test owns
    x = big[:8]
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert eng.lib.b2m_check_errors(eng._h, stream) == 0
    assert eng.lib.b2m_set_input_perm(eng._h, 0, C.c_void_p(dev.data_ptr())) == 0
    eng.route(0, x)
    assert eng.lib.b2m_check_errors(eng._h, stream) == L.B2M_EINVAL
    assert b"input-permutation" in eng.lib.b2m_last_error(eng._h)
    xp = eng.ws("xp", 8)[:16]
    assert bool((xp[:, 7] == 0).all())
    assert eng.lib.b2m_check_errors(eng._h, stream) == 0          # the report cleared the sticky word
    eng.set_input_perm(0, None)
    eng.route(0, x)
    assert eng.lib.b2m_check_errors(eng._h, stream) == 0
    eng.close()
