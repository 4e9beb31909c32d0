"""GPU: the decode GEMMs reading experts from the 12-bit packed copy (csrc/weight_pack.cuh) give bit-identical results.

Every check compares an engine with the packed copy (MoEEngine default) against the same weights in an engine that reads the
bf16 slots only (pack_weights=False): full-size Mixtral layers at T = 1, 8, 64 with bench-style and adversarial weights
(patched and uncodable tiles), rewriting experts through load_expert, a graph captured while slots are stale, a
DeepSeek-V2-Lite-shaped layer, and an offload context (which must not allocate the copy).  The second eager forward of a layer
after its experts were written packs them: the tests warm up twice before they compare."""
import pytest
import torch

pytestmark = pytest.mark.gpu

H, I, E, K = 4096, 14336, 8, 2
DT = torch.bfloat16


def _engine(pack, H=H, I=I, E=E, K=K, L=1, **kw):
    from moe_infinity_b200 import MoEEngine
    return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=64, pack_weights=pack, **kw)


def _weights(seed, H=H, I=I, E=E, adversarial=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ws = []
    for e in range(E):
        w = [(torch.randn(I, H, generator=g, device="cuda") * 0.02).to(DT),
             (torch.randn(H, I, generator=g, device="cuda") * 0.02).to(DT),
             (torch.randn(I, H, generator=g, device="cuda") * 0.02).to(DT)]
        if adversarial:
            w1, w2, w3 = w
            for r in range(0, 128, 16):
                w1[r, (r * 7) % 64] = 3e-9                             # a few values below the window: patched tile
            for r in range(128, 256, 6):
                w1[r, 64 + (r * 5) % 64] = -4e-9                       # 22 of them: the tile cannot be coded
            w2[0:8, 0:64] = 0.0                                        # +0 rows
            w2[8:16, 0:64] = -0.0                                      # -0 rows
            w2[256, 133] = 1e-40                                       # a subnormal: patched
            if e % 2:
                w3[384, 640] = 70000.0                                 # window above 2^15: this matrix stays bf16
        ws.append(w)
    return ws


def _load(eng, ws, layer=0):
    for e, w in enumerate(ws):
        eng.load_expert(layer, e, w)


def _pair(ws, gate):
    a, b = _engine(True), _engine(False)
    for eng in (a, b):
        _load(eng, ws)
        eng.set_gate(0, gate)
    return a, b


def _fwd(eng, x, **kw):
    out = eng.forward(0, x, **kw)
    torch.cuda.synchronize()
    return out.clone()


@pytest.mark.parametrize("adversarial", [False, True], ids=["bench_weights", "adversarial"])
def test_packed_matches_bf16_fullsize(adversarial, lib_built):
    ws = _weights(1, adversarial=adversarial)
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    a, b = _pair(ws, gate)
    free0 = torch.cuda.mem_get_info()[0]
    x = torch.randn(8, H, device="cuda").to(DT)
    assert torch.equal(_fwd(a, x), _fwd(b, x))    # first forward after the load: bf16 in both
    assert torch.equal(_fwd(a, x), _fwd(b, x))    # second: the packed engine packs, then reads the packed copy
    for T in (1, 8, 64):
        x = torch.randn(T, H, device="cuda").to(DT)
        ya, yb = _fwd(a, x), _fwd(b, x)
        assert torch.equal(ya, yb), f"T={T}: packed and bf16 engines differ"
        assert torch.isfinite(yb.float()).all()
    # the packed engine allocated its copy on the first forward (0.76 of 2.8 GB)
    assert free0 - torch.cuda.mem_get_info()[0] > 1.5e9
    a.close(); b.close()


def test_rewrite_through_load_expert(lib_built):
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    x = torch.randn(8, H, device="cuda").to(DT)
    eng = _engine(True)
    _load(eng, _weights(2))
    eng.set_gate(0, gate)
    _fwd(eng, x); _fwd(eng, x)            # packs the first weights
    new = _weights(3)
    _load(eng, new)                       # same slots, new weights: stale until the second forward packs them again
    got1, got = _fwd(eng, x), _fwd(eng, x)
    fresh = _engine(True)
    _load(fresh, new)
    fresh.set_gate(0, gate)
    _fwd(fresh, x)
    ref = _fwd(fresh, x)
    bf = _engine(False)
    _load(bf, new)
    bf.set_gate(0, gate)
    assert torch.equal(got, ref) and torch.equal(got1, ref) and torch.equal(got, _fwd(bf, x))
    for e_ in (eng, fresh, bf):
        e_.close()


def test_graph_captured_while_stale(lib_built):
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    x = torch.randn(8, H, device="cuda").to(DT)
    eng = _engine(True)
    _load(eng, _weights(4))
    eng.set_gate(0, gate)
    _fwd(eng, x); _fwd(eng, x)            # eager: routing row uploaded, slots packed
    new = _weights(5)
    _load(eng, new)                       # stale: a capture now must read the bf16 slots
    ref_eng = _engine(False)
    _load(ref_eng, new)
    ref_eng.set_gate(0, gate)
    ref = _fwd(ref_eng, x)
    out = torch.empty_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.forward(0, x, out=out)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    _fwd(eng, x); _fwd(eng, x)            # eager forwards pack; the graph now reads the packed copy (flags are device state)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    eng.close(); ref_eng.close()


def test_deepseek_lite_shape(lib_built):
    from moe_infinity_b200 import _lib as L
    Hd, Id, Ed, Kd = 2048, 1408, 64, 6
    ws = _weights(6, H=Hd, I=Id, E=Ed)
    ws = [[w[0], w[2], w[1]] for w in ws]   # gate | up | down
    logits = torch.randn(64, Ed, device="cuda").to(DT)
    outs = []
    for pack in (True, False):
        eng = _engine(pack, H=Hd, I=Id, E=Ed, K=Kd, expert_type=L.EXPERT_DEEPSEEK)
        _load(eng, ws)
        res = []
        for T in (1, 1, 16, 64):
            x = torch.randn(T, Hd, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
            res.append(_fwd(eng, x, router_logits=logits[:T]))
        outs.append(res)
        eng.close()
    for T, ya, yb in zip((1, 1, 16, 64), *outs):
        assert torch.equal(ya, yb), f"T={T}"


def test_offload_context_has_no_packed_copy(lib_built):
    Hs, Is, Es = 1024, 2048, 8
    ws = _weights(7, H=Hs, I=Is, E=Es)
    from moe_infinity_b200 import MoEEngine
    eng = MoEEngine(num_layers=2, num_experts=Es, hidden=Hs, inter=Is, top_k=2, dtype=DT, max_tokens=64, num_slots=Es)
    cpu = [[t.cpu() for t in w] for w in ws]
    for l in range(2):
        for e in range(Es):
            eng.register_expert(l, e, cpu[e])
    x = torch.randn(8, Hs, device="cuda").to(DT)
    logits = torch.randn(8, Es, device="cuda").to(DT)
    out = torch.empty_like(x)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        for l in range(2):
            eng.forward(l, x, router_logits=logits, out=out)
    torch.cuda.synchronize()
    shadow = Es * 3 * Hs * Is * 2 * 0.75
    assert free0 - torch.cuda.mem_get_info()[0] < shadow / 4
    eng.close()
