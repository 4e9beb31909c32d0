"""GPU: routed experts stored as 4-bit integers with an fp16 scale and zero point per 128 inputs, run with f16 activations
(MoEEngine(dtype=torch.float16, expert_dtype=torch.uint4): B2M_WEIGHTS_INT4_G128_F16, the AWQ / GPTQ format).

Every check compares a format-6 engine with an f16 engine (pack_weights=False) loaded with `dequantize_g128(q, s, z,
torch.float16)` of the same codes, scales and zero points, and demands torch.equal.  Where the f16 engine itself does not
reproduce its output (fp32 atomics of a down projection split over three or more CTAs, or of the f16 shared expert),
`_check_same` holds the gate/up output to torch.equal and the layer output to the existing 2-ulp bound, as the bf16 int4
tests do.  Covered: a full-size Mixtral layer from T=1 to 1024 with quantised N(0, 0.02) and adversarial weights (every
(q, z) pair, fp16-subnormal products, negative scales, an all-zero group; products kept finite), a DeepSeek-V2-Lite shaped
layer with f16 shared experts, a DeepSeek-V3 routed layer, rewritten HBM-only experts, host-backed experts in an offload
context with fewer slots than active experts, a captured DecodeSession, synthetic AWQ and GPTQ checkpoints loaded through
hf.load_int4_checkpoint, and hf.patch_mixtral on a tiny f16 Mixtral."""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

H, I, E, K = 4096, 14336, 8, 2
DT = torch.float16
U4 = torch.uint4


def _engine(int4, H=H, I=I, E=E, K=K, L=1, max_tokens=1024, **kw):
    from moe_infinity_b200 import MoEEngine
    if int4:
        return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                         expert_dtype=U4, **kw)
    return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                     pack_weights=False, **kw)


def _adversarial(q, s, z):
    """Rows 0..127, group 0: codes 0..15 along the row and z = row % 16 -- every (q, z) pair.  Rows 0..127, other groups:
    scales from 2^-24 to 2^-4, a third of them negative (|W| <= 1.5, so every GEMM output stays finite in f16).  Rows
    128..255: fp16 subnormal scales (+-), so every product is an fp16 subnormal or +-0.  Rows 256..383, group 1: an all-zero
    group (codes = zero point = 0)."""
    dev = q.device
    c = torch.arange(128, device=dev) % 16
    q[:128, :64] = (c[0::2] | (c[1::2] << 4)).to(torch.uint8)[None, :]
    z[:128, 0] = (torch.arange(128, device=dev) % 16).to(torch.uint8)
    r = torch.arange(128, device=dev)[:, None]
    g = torch.arange(s.shape[1], device=dev)[None, :]
    v = torch.exp2(((r * 7 + g * 3) % 21 - 24).float()) * (1 + ((r + g) % 5).float() / 7)
    s[:128] = torch.where((r + g) % 3 == 0, -v, v).to(DT)
    bits = ((torch.arange(128, device=dev)[:, None] * 5 + g * 11) % 1023 + 1).to(torch.int16)
    bits = torch.where((r + g) % 2 == 0, bits, bits | -0x8000)
    s[128:256] = bits.view(DT)
    q[256:384, 64:128] = 0
    z[256:384, 1] = 0
    return q, s, z


def _int4_weights(seed, H=H, I=I, E=E, shapes=None, adversarial=False):
    """[(q list, s list, z list)] per expert from quantize_g128(scale_dtype=float16) of N(0, 0.02)."""
    from moe_infinity_b200.int4 import quantize_g128
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = shapes or [(I, H), (H, I), (I, H)]
    out = []
    for e in range(E):
        qs, ss, zs = [], [], []
        for m, shp in enumerate(shapes):
            q, s, z = quantize_g128(torch.randn(*shp, generator=g, device="cuda") * 0.02, scale_dtype=DT)
            if adversarial and m != 2 and e % 2 == 0:
                q, s, z = _adversarial(q, s, z)
            qs.append(q); ss.append(s); zs.append(z)
        out.append((qs, ss, zs))
    return out


def _deq(ws):
    from moe_infinity_b200.int4 import dequantize_g128
    return [[dequantize_g128(q, s, z, DT) for q, s, z in zip(*ex)] for ex in ws]


def _load_pair(a, b, ws, layer=0):
    for e, ((qs, ss, zs), w) in enumerate(zip(ws, _deq(ws))):
        a.load_expert(layer, e, qs, scales=ss, zeros=zs)
        b.load_expert(layer, e, w)


def _fwd(eng, x, layer=0, **kw):
    out = eng.forward(layer, x, **kw)
    torch.cuda.synchronize()
    return out.clone()


def _fwd_ws(eng, x, layer=0, **kw):
    out = _fwd(eng, x, layer, **kw)
    T = x.shape[0]
    return out, eng.ws("hmid", T).clone(), eng.ws("y", T).clone()


def _check_same(a, b, x, what, layer=0, **kw):
    """The format-6 engine `a` against the f16 engine `b` on one input: gate/up outputs bit for bit; the routed experts'
    fp32 outputs bit for bit whenever both engines reproduce their own; the layer outputs bit for bit or, where split-K
    atomics or the shared expert make the f16 engine itself nondeterministic, within hidden_close's 2-ulp bound."""
    from test_gpu_parity import hidden_close
    oa, ha, ya = _fwd_ws(a, x, layer, **kw)
    _, _, ya2 = _fwd_ws(a, x, layer, **kw)
    ob, hb, yb = _fwd_ws(b, x, layer, **kw)
    _, _, yb2 = _fwd_ws(b, x, layer, **kw)
    assert torch.isfinite(ha.float()).all() and torch.isfinite(oa.float()).all(), f"{what}: non-finite outputs"
    assert torch.equal(ha, hb), f"{what}: gate/up outputs differ"
    if torch.equal(ya, ya2) and torch.equal(yb, yb2):
        assert torch.equal(ya, yb), f"{what}: routed expert outputs differ ({(ya - yb).abs().max().item()})"
    if not torch.equal(oa, ob):
        hidden_close(oa, ob.cpu(), None, DT, what)


def test_adversarial_groups_cover_the_edges():
    from moe_infinity_b200.int4 import dequantize_g128, unpack_codes
    (qs, ss, zs), = _int4_weights(5, H=1024, I=2048, E=1, adversarial=True)
    q, s, z = qs[0], ss[0], zs[0]
    codes = unpack_codes(q[:128, :64]).long()
    assert len(set((codes * 16 + z[:128, :1].long()).flatten().tolist())) == 256
    w = dequantize_g128(q, s, z, DT)
    bits = w.view(torch.int16).int() & 0xffff
    sub = ((bits & 0x7c00) == 0) & ((bits & 0x3ff) != 0)
    assert bool(sub[128:256].any()) and bool((s.float() < 0).any()) and bool(torch.isfinite(w.float()).all())
    assert bool((bits[256:384, 128:256] == 0).all())


@pytest.mark.parametrize("adversarial", [False, True], ids=["normal_weights", "adversarial"])
def test_int4_f16_matches_f16_fullsize(adversarial, lib_built):
    from moe_infinity_b200.int4 import expert_blob_bytes
    ws = _int4_weights(1, adversarial=adversarial)
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    a, b = _engine(True), _engine(False)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.set_gate(0, gate)
    assert a.stats()["slot_bytes"] == expert_blob_bytes(H, I) == 93585408
    for T in (1, 8, 16, 64, 128, 256, 1024):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        for _ in range(2):
            _check_same(a, b, x, f"T={T}")
        if not adversarial:
            assert _fwd(a, x).float().abs().max() > 0
    a.close(); b.close()


def test_deepseek_lite_shape(lib_built):
    from moe_infinity_b200 import _lib as L
    Hd, Id, Ed, Kd, Is = 2048, 1408, 64, 6, 2816
    ws = _int4_weights(6, H=Hd, I=Id, E=Ed, shapes=[(Id, Hd), (Id, Hd), (Hd, Id)])   # gate | up | down
    g = torch.Generator(device="cuda").manual_seed(60)
    shared = [(torch.randn(Is, Hd, generator=g, device="cuda") * 0.02).to(DT),
              (torch.randn(Is, Hd, generator=g, device="cuda") * 0.02).to(DT),
              (torch.randn(Hd, Is, generator=g, device="cuda") * 0.02).to(DT)]
    gate = torch.randn(Ed, Hd, generator=g, device="cuda") * 0.05
    kw = dict(H=Hd, I=Id, E=Ed, K=Kd, max_tokens=512, expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_GROUP,
              n_group=8, topk_group=3, shared_inter=Is)
    a, b = _engine(True, **kw), _engine(False, **kw)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.register_shared(0, shared)
        eng.set_gate(0, gate)
    for T in (1, 8, 512):
        x = torch.randn(T, Hd, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        _check_same(a, b, x, f"T={T}")
    a.close(); b.close()


def test_deepseek_v3_routed_layer(lib_built):
    """A V3-routed layer (E=256, k=8, 8 groups keep 4, correction bias, one f16 shared expert) at reduced H and I."""
    from moe_infinity_b200 import _lib as L
    Hv, Iv, Ev, Kv = 1024, 256, 256, 8
    ws = _int4_weights(7, H=Hv, I=Iv, E=Ev, shapes=[(Iv, Hv), (Iv, Hv), (Hv, Iv)])
    g = torch.Generator(device="cuda").manual_seed(70)
    shared = [(torch.randn(shp, generator=g, device="cuda") * 0.02).to(DT) for shp in ((Iv, Hv), (Iv, Hv), (Hv, Iv))]
    gate = torch.randn(Ev, Hv, generator=g, device="cuda") * (1.0 / Hv ** 0.5)
    bias = torch.randn(Ev, generator=g, device="cuda") * 0.1
    kw = dict(H=Hv, I=Iv, E=Ev, K=Kv, max_tokens=256, expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_V3,
              n_group=8, topk_group=4, norm_topk_prob=True, routed_scaling_factor=2.5, shared_inter=Iv,
              gate_dtype=torch.float32)
    a, b = _engine(True, **kw), _engine(False, **kw)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.register_shared(0, shared)
        eng.set_gate(0, gate)
        eng.set_gate_bias(0, bias)
    for T in (1, 8, 64, 256):
        x = torch.randn(T, Hv, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        _check_same(a, b, x, f"T={T}")
    a.close(); b.close()


def test_rewrite_and_offload(lib_built):
    Hs, Is, Es = 1024, 2048, 8
    gate = (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT)
    x = torch.randn(8, Hs, device="cuda").to(DT)
    a, b = _engine(True, H=Hs, I=Is, E=Es), _engine(False, H=Hs, I=Is, E=Es)
    _load_pair(a, b, _int4_weights(2, H=Hs, I=Is, E=Es))
    for eng in (a, b):
        eng.set_gate(0, gate)
    _check_same(a, b, x, "first weights")
    _load_pair(a, b, _int4_weights(3, H=Hs, I=Is, E=Es))
    _check_same(a, b, x, "rewritten weights")
    a.close(); b.close()
    # host-backed experts, 3 slots for 2 layers x 8 experts: every layer call runs in waves, evicts and re-stages
    ws = [_int4_weights(10 + l, H=Hs, I=Is, E=Es) for l in range(2)]
    a = _engine(True, H=Hs, I=Is, E=Es, L=2, num_slots=3, max_tokens=64)
    b = _engine(False, H=Hs, I=Is, E=Es, L=2, num_slots=3, max_tokens=64)
    for l in range(2):
        for e, ((qs, ss, zs), w) in enumerate(zip(ws[l], _deq(ws[l]))):
            a.register_expert(l, e, [q.cpu() for q in qs], scales=[s.cpu() for s in ss], zeros=[z.cpu() for z in zs])
            b.register_expert(l, e, [t.cpu() for t in w])
    logits = torch.randn(16, Es, device="cuda").to(DT)
    for step in range(2):
        for l in range(2):
            xl = torch.randn(16, Hs, device="cuda", generator=torch.Generator(device="cuda").manual_seed(10 * step + l)).to(DT)
            _check_same(a, b, xl, f"step {step} layer {l}", l, router_logits=logits)
    sa = a.stats()
    assert sa["misses"] > 6 and sa["evictions"] > 0
    assert sa["h2d_bytes"] == sa["misses"] * a.expert_bytes and a.expert_bytes < 0.27 * b.expert_bytes
    a.close(); b.close()


def test_scale_dtype_must_match_engine(lib_built):
    """Scales of the other 16-bit type are refused, never rounded."""
    Hs, Is, Es = 1024, 2048, 2
    (qs, ss, zs), = _int4_weights(4, H=Hs, I=Is, E=1)
    a = _engine(True, H=Hs, I=Is, E=Es, K=1, max_tokens=16)
    with pytest.raises(ValueError, match="float16"):
        a.load_expert(0, 0, qs, scales=[s.to(torch.bfloat16) for s in ss], zeros=zs)
    a.close()
    from moe_infinity_b200 import MoEEngine
    b = MoEEngine(num_layers=1, num_experts=Es, hidden=Hs, inter=Is, top_k=1, dtype=torch.bfloat16, max_tokens=16,
                  expert_dtype=U4)
    with pytest.raises(ValueError, match="bfloat16"):
        b.load_expert(0, 0, qs, scales=ss, zeros=zs)
    b.close()


def test_decode_session_graph(lib_built):
    from moe_infinity_b200 import DecodeSession
    Hs, Is, Es, T = 1024, 2048, 8, 8
    a = _engine(True, H=Hs, I=Is, E=Es, L=2, max_tokens=64)
    for l in range(2):
        for e, (qs, ss, zs) in enumerate(_int4_weights(20 + l, H=Hs, I=Is, E=Es)):
            a.load_expert(l, e, qs, scales=ss, zeros=zs)
        a.set_gate(l, (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT))
    sess = DecodeSession(a, T)
    sess.x_host.copy_(torch.randn(2, T, Hs).to(DT))
    eager = torch.stack([_fwd(a, sess.x_host[l].cuda(), l) for l in range(2)]).cpu()
    sess.capture()
    out = sess.step().clone()
    assert torch.equal(out, eager)
    a.close()


def _checkpoint_pair(tmp_path, method):
    """A synthetic 2-layer checkpoint in `method`'s layout and the weights it holds, dequantised the test's own way."""
    import int4_checkpoint_packers as P
    g = torch.Generator().manual_seed(11)
    tensors, deq = {}, {}
    if method == "awq":                      # Mixtral layout
        Lc, Ec, Hc, Ic, names, moe = 2, 8, 1024, 2048, ("w1", "w2", "w3"), "block_sparse_moe"
        shapes = ((Ic, Hc), (Hc, Ic), (Ic, Hc))
    else:                                    # DeepSeek layout, layer 0 dense, f16 shared experts
        Lc, Ec, Hc, Ic, names, moe = 2, 16, 1024, 512, ("gate_proj", "up_proj", "down_proj"), "mlp"
        shapes = ((Ic, Hc), (Ic, Hc), (Hc, Ic))
        tensors["model.layers.0.mlp.gate_proj.weight"] = torch.zeros(8, 8, dtype=DT)

    def put(pre, o, i):
        q, s, z = P.random_qsz(o, i, g, z_lo=1, s_std=0.0015)
        if method == "awq":
            qw, qz, sc = P.awq_pack(q, s, z)
            tensors.update({f"{pre}.qweight": qw, f"{pre}.qzeros": qz, f"{pre}.scales": sc})
        else:
            qw, qz, sc, gi = P.gptq_pack(q, s, z)
            tensors.update({f"{pre}.qweight": qw, f"{pre}.qzeros": qz, f"{pre}.scales": sc, f"{pre}.g_idx": gi})
        deq[pre] = P.fp16_dequant(q, s, z)

    layers = [0, 1] if method == "awq" else [1]
    for l in layers:
        base = f"model.layers.{l}.{moe}"
        tensors[f"{base}.gate.weight"] = (torch.randn(Ec, Hc, generator=g) * 0.05).to(DT)
        for e in range(Ec):
            for n, (o, i) in zip(names, shapes):
                put(f"{base}.experts.{e}.{n}", o, i)
        if method != "awq":
            for n, (o, i) in zip(names, ((Ic, Hc), (Ic, Hc), (Hc, Ic))):
                put(f"{base}.shared_experts.{n}", o, i)
    shards = P.write_shards(str(tmp_path), tensors)
    return shards, tensors, deq, (Lc, Ec, Hc, Ic, names, moe, layers)


@pytest.mark.parametrize("method", ["awq", "gptq"])
def test_load_int4_checkpoint(tmp_path, method, lib_built):
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200.hf import load_int4_checkpoint
    shards, tensors, deq, (Lc, Ec, Hc, Ic, names, moe, layers) = _checkpoint_pair(tmp_path, method)
    if method == "awq":
        kw = dict(H=Hc, I=Ic, E=Ec, K=2, L=Lc, max_tokens=128)
        cfg = dict(quant_method="awq", bits=4, group_size=128, zero_point=True, version="gemm")
        mtype = "mixtral"
    else:
        kw = dict(H=Hc, I=Ic, E=Ec, K=4, L=Lc, max_tokens=128, expert_type=L.EXPERT_DEEPSEEK,
                  router=L.ROUTER_DEEPSEEK_GREEDY, shared_inter=Ic)
        cfg = dict(quant_method="gptq", bits=4, group_size=128, desc_act=False, checkpoint_format="gptq")
        mtype = "deepseek_v2"
    a, b = _engine(True, **kw), _engine(False, **kw)
    assert load_int4_checkpoint(a, shards, cfg, mtype) == layers
    for l in layers:
        base = f"model.layers.{l}.{moe}"
        for e in range(Ec):
            b.load_expert(l, e, [deq[f"{base}.experts.{e}.{n}"].cuda() for n in names])
        if method != "awq":
            b.register_shared(l, [deq[f"{base}.shared_experts.{n}"] for n in names])
        b.set_gate(l, tensors[f"{base}.gate.weight"])
    for l in layers:
        for T in (8, 128):
            x = torch.randn(T, Hc, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T + l)).to(DT)
            _check_same(a, b, x, f"{method} layer {l} T={T}", l)
    a.close(); b.close()


def test_patched_mixtral_int4_f16(lib_built):
    """hf.patch_mixtral on an f16 model with an f16 int4 engine against the same patch with an f16 engine holding the
    dequantised weights."""
    from moe_infinity_b200.hf import patch_mixtral
    from moe_infinity_b200.int4 import dequantize_g128, quantize_g128
    from test_gpu_hf_mixtral import _tiny
    ref = _tiny().to(DT)
    cfg = ref.config
    Lm, Em, Hm, Im = cfg.num_hidden_layers, cfg.num_local_experts, cfg.hidden_size, cfg.intermediate_size
    deq = copy.deepcopy(ref)
    with torch.no_grad():   # the f16 model holds what the int4 engine computes with
        for layer in deq.model.layers:
            ex = layer.mlp.experts
            for e in range(Em):
                for p, rows in ((ex.gate_up_proj, slice(0, Im)), (ex.gate_up_proj, slice(Im, 2 * Im)), (ex.down_proj, slice(None))):
                    p.data[e, rows] = dequantize_g128(*quantize_g128(p.data[e, rows], scale_dtype=DT), DT)
    a = _engine(True, H=Hm, I=Im, E=Em, K=cfg.num_experts_per_tok, L=Lm, max_tokens=256)
    ours = copy.deepcopy(ref)
    patch_mixtral(ours, engine=a)
    b = _engine(False, H=Hm, I=Im, E=Em, K=cfg.num_experts_per_tok, L=Lm, max_tokens=256)
    patch_mixtral(deq, engine=b)
    ids = torch.randint(0, cfg.vocab_size, (2, 24), device="cuda")
    with torch.no_grad():
        la = ours(ids).logits
        lb = deq(ids).logits
        lb2 = deq(ids).logits
    if torch.equal(lb, lb2):
        assert torch.equal(la, lb)
    else:
        rms = lb.float().pow(2).mean().sqrt()
        assert (la.float() - lb.float()).abs().max() <= 0.02 * rms and (la.argmax(-1) == lb.argmax(-1)).float().mean() > 0.97
    assert a.stats()["slot_bytes"] < 0.27 * b.stats()["slot_bytes"]
