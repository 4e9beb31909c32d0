"""GPU: routed experts stored as FP8 E4M3 with 128x128 block scales (MoEEngine(expert_dtype=torch.float8_e4m3fn)).

Every check compares an fp8 engine with a bf16 engine (pack_weights=False) loaded with `dequantize_block128` of the same
e4m3 weights and scales, and demands torch.equal: the fp8 GEMMs dequantise inside the kernel with exactly the documented
roundings and keep the bf16 engine's launch plan.  (Where the bf16 engine itself does not reproduce its output -- fp32
atomics of a down projection split over three or more CTAs, or of a bf16 shared expert -- `_check_same` says what is held.)  Covered: a full-size Mixtral layer from decode to prefill (16..128-token
gate/up tiles, split-K / stream-K, dual_m, 256-token down tiles) with N(0, 0.02) and adversarial weights, a DeepSeek-V2-Lite
shaped layer with bf16 shared experts, rewritten HBM-only experts, host-backed experts in an offload context with fewer slots
than active experts, a captured DecodeSession, the absence of the 12-bit packed copy, and the CPU oracle at a small size."""
import pytest
import torch

pytestmark = pytest.mark.gpu

H, I, E, K = 4096, 14336, 8, 2
DT = torch.bfloat16
FP8 = torch.float8_e4m3fn


def _engine(fp8, H=H, I=I, E=E, K=K, L=1, max_tokens=1024, **kw):
    from moe_infinity_b200 import MoEEngine
    if fp8:
        return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                         expert_dtype=FP8, **kw)
    return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                     pack_weights=False, **kw)


def _adversarial(q, s):
    """Every finite e4m3 code (+-0 and subnormals included) in block (0, 0), an all-zero block (1, 1), and block scales
    spanning 2^-30 .. 2^10."""
    codes = torch.tensor([c for c in range(256) if c & 0x7f != 0x7f], dtype=torch.uint8, device=q.device)
    qb = q.view(torch.uint8)
    qb[:128, :128] = codes.repeat(128 * 128 // len(codes) + 1)[:128 * 128].view(128, 128)
    qb[128:256, 128:256] = 0
    r = torch.arange(s.shape[0], device=s.device)[:, None]
    c = torch.arange(s.shape[1], device=s.device)[None, :]
    s.copy_(torch.exp2(((r * 7 + c * 3) % 41 - 30).float()) * (1 + ((r + c) % 5).float() / 7))
    s[1, 1] = 1.0
    return q, s


def _fp8_weights(seed, H=H, I=I, E=E, shapes=None, adversarial=False):
    """[(w_q list, s list)] per expert from quantize_block128 of N(0, 0.02)."""
    from moe_infinity_b200.fp8 import quantize_block128
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = shapes or [(I, H), (H, I), (I, H)]
    out = []
    for e in range(E):
        qs, ss = [], []
        for m, shp in enumerate(shapes):
            q, s = quantize_block128(torch.randn(*shp, generator=g, device="cuda") * 0.02)
            if adversarial and m != 2 and e % 2 == 0:
                q, s = _adversarial(q, s)
            qs.append(q); ss.append(s)
        out.append((qs, ss))
    return out


def _deq(ws):
    from moe_infinity_b200.fp8 import dequantize_block128
    return [[dequantize_block128(q, s) for q, s in zip(qs, ss)] for qs, ss in ws]


def _load_pair(a, b, ws, layer=0):
    for e, ((qs, ss), w) in enumerate(zip(ws, _deq(ws))):
        a.load_expert(layer, e, qs, scales=ss)
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
    """The fp8 engine `a` against the bf16 engine `b` on one input.  The gate/up GEMM (no split-K) must agree bit for bit.
    The routed experts' fp32 outputs must too whenever the bf16 engine reproduces its own: a down projection split over three
    or more CTAs (small or partial waves) adds its fp32 partials with atomics in arrival order, and then two runs of the SAME
    engine may differ in the last bit -- as may a bf16 shared expert's output.  Only those are held to hidden_close's 2-ulp
    bound instead."""
    from test_gpu_parity import hidden_close
    oa, ha, ya = _fwd_ws(a, x, layer, **kw)
    ob, hb, yb = _fwd_ws(b, x, layer, **kw)
    _, _, yb2 = _fwd_ws(b, x, layer, **kw)
    assert torch.equal(ha, hb), f"{what}: gate/up outputs differ"
    if torch.equal(yb, yb2):
        assert torch.equal(ya, yb), f"{what}: routed expert outputs differ ({(ya - yb).abs().max().item()})"
    if not torch.equal(oa, ob):
        hidden_close(oa, ob.cpu(), None, DT, what)


@pytest.mark.parametrize("adversarial", [False, True], ids=["normal_weights", "adversarial"])
def test_fp8_matches_bf16_fullsize(adversarial, lib_built):
    from moe_infinity_b200.fp8 import expert_blob_bytes
    ws = _fp8_weights(1, adversarial=adversarial)
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    a, b = _engine(True), _engine(False)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.set_gate(0, gate)
    assert a.stats()["slot_bytes"] == expert_blob_bytes(H, I) == 176203776
    for T in (1, 8, 64, 200, 1024):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        for _ in range(2):   # (a bf16 engine with the packed copy would change path on the second forward; neither does)
            ya, yb = _fwd(a, x), _fwd(b, x)
            assert torch.equal(ya, yb), f"T={T}: fp8 and bf16 engines differ ({(ya.float() - yb.float()).abs().max().item()})"
        if not adversarial:
            assert torch.isfinite(ya.float()).all() and ya.float().abs().max() > 0
    a.close(); b.close()


def test_deepseek_lite_shape(lib_built):
    from moe_infinity_b200 import _lib as L
    Hd, Id, Ed, Kd, Is = 2048, 1408, 64, 6, 2816
    ws = _fp8_weights(6, H=Hd, I=Id, E=Ed, shapes=[(Id, Hd), (Id, Hd), (Hd, Id)])   # gate | up | down
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


def test_rewrite_and_offload(lib_built):
    Hs, Is, Es = 1024, 2048, 8
    gate = (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT)
    x = torch.randn(8, Hs, device="cuda").to(DT)
    # HBM-only experts, rewritten in place through load_expert
    a, b = _engine(True, H=Hs, I=Is, E=Es), _engine(False, H=Hs, I=Is, E=Es)
    _load_pair(a, b, _fp8_weights(2, H=Hs, I=Is, E=Es))
    for eng in (a, b):
        eng.set_gate(0, gate)
    _check_same(a, b, x, "first weights")
    _load_pair(a, b, _fp8_weights(3, H=Hs, I=Is, E=Es))
    _check_same(a, b, x, "rewritten weights")
    a.close(); b.close()
    # host-backed experts, 3 slots for 2 layers x 8 experts: every layer call runs in waves, evicts and re-stages
    ws = [_fp8_weights(10 + l, H=Hs, I=Is, E=Es) for l in range(2)]
    a = _engine(True, H=Hs, I=Is, E=Es, L=2, num_slots=3, max_tokens=64)
    b = _engine(False, H=Hs, I=Is, E=Es, L=2, num_slots=3, max_tokens=64)
    for l in range(2):
        for e, ((qs, ss), w) in enumerate(zip(ws[l], _deq(ws[l]))):
            a.register_expert(l, e, [q.cpu() for q in qs], scales=[s.cpu() for s in ss])
            b.register_expert(l, e, [t.cpu() for t in w])
    logits = torch.randn(16, Es, device="cuda").to(DT)
    for step in range(2):
        for l in range(2):
            xl = torch.randn(16, Hs, device="cuda", generator=torch.Generator(device="cuda").manual_seed(10 * step + l)).to(DT)
            _check_same(a, b, xl, f"step {step} layer {l}", l, router_logits=logits)
    sa, sb = a.stats(), b.stats()
    assert sa["misses"] > 6 and sa["evictions"] > 0
    assert sa["h2d_bytes"] == sa["misses"] * a.expert_bytes and a.expert_bytes < 0.501 * b.expert_bytes
    a.close(); b.close()


def test_decode_session_graph(lib_built):
    from moe_infinity_b200 import DecodeSession
    Hs, Is, Es, T = 1024, 2048, 8, 8
    a = _engine(True, H=Hs, I=Is, E=Es, L=2, max_tokens=64)
    for l in range(2):
        for e, (qs, ss) in enumerate(_fp8_weights(20 + l, H=Hs, I=Is, E=Es)):
            a.load_expert(l, e, qs, scales=ss)
        a.set_gate(l, (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT))
    sess = DecodeSession(a, T)
    sess.x_host.copy_(torch.randn(2, T, Hs).to(DT))
    eager = torch.stack([_fwd(a, sess.x_host[l].cuda(), l) for l in range(2)]).cpu()
    sess.capture()
    out = sess.step().clone()
    assert torch.equal(out, eager)
    a.close()


def test_no_packed_copy(lib_built):
    Hs, Is, Es = 2048, 4096, 8
    a = _engine(True, H=Hs, I=Is, E=Es, max_tokens=64)
    for e, (qs, ss) in enumerate(_fp8_weights(30, H=Hs, I=Is, E=Es)):
        a.load_expert(0, e, qs, scales=ss)
    a.set_gate(0, (torch.randn(Es, Hs, device="cuda") * 0.05).to(DT))
    x = torch.randn(8, Hs, device="cuda").to(DT)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        _fwd(a, x)
    shadow = Es * 3 * Hs * Is * 2 * 0.75   # what a bf16 context's packed copy of these experts would take
    assert free0 - torch.cuda.mem_get_info()[0] < shadow / 4
    a.close()


def test_against_cpu_oracle(lib_built):
    from test_gpu_parity import hidden_close
    from moe_infinity_b200.fp8 import dequantize_block128, quantize_block128
    from oracle import moe_oracle as O
    Hs, Is, Es, k, T = 256, 512, 8, 2, 24
    experts = O.make_experts(Es, Hs, Is, torch.float32, seed=3, std=0.05)
    q = [[quantize_block128(w) for w in ex] for ex in experts]
    deq = [[dequantize_block128(wq, s) for wq, s in ex] for ex in q]
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, T, Hs, generator=g).to(DT)
    gate = (torch.randn(Es, Hs, generator=g) * 0.1).to(DT)
    ref, logits, _ = O.mixtral_block(x, gate, deq, k)
    a = _engine(True, H=Hs, I=Is, E=Es, K=k, max_tokens=64)
    for e, ex in enumerate(q):
        a.load_expert(0, e, [wq for wq, _ in ex], scales=[s for _, s in ex])
    a.set_gate(0, gate)
    out = _fwd(a, x.cuda(), router_logits=logits.cuda())
    hidden_close(out, ref, None, DT, "fp8 experts vs the CPU oracle on the dequantised weights")
    a.close()
