"""GPU: routed experts stored as FP8 E4M3 with one fp32 scale per output channel
(MoEEngine(expert_dtype=torch.float8_e4m3fn, fp8_scales="row"), B2M_WEIGHTS_FP8_E4M3_ROW).

Every check holds the row-format engine to a bf16 engine (pack_weights=False) loaded with `dequantize_row` of the same
codes and scales, under torch.equal -- except where the bf16 engine does not reproduce its own output (fp32 atomics of a
down projection split over three or more CTAs, or of a bf16 shared expert), where the helpers of the block-format and
Llama 4 tests say what is held.  Covered: a full-size Mixtral layer at T = 1 .. 1024 (decode tiles, prefill, split-K,
dual_m) with N(0, 0.02) and adversarial weights, the DeepSeek-V3 router with a shared expert, Qwen3-MoE, Llama 4 with its
shared expert, offload, a captured decode graph; every fp8 launch plan of tests/gemm_exact_cases.py against its float64
reference; and hf.load_fp8_checkpoint end to end: a tiny Llama 4 FP8 checkpoint into patch_llama4's engine against a bf16
model holding the dequantised experts, and Qwen3-MoE / DeepSeek-V3 block-FP8 checkpoints against a block engine fed the
same tensors by hand."""
from __future__ import annotations

import copy

import pytest
import torch
import torch.nn.functional as F

import gemm_exact_cases as X
from int4_checkpoint_packers import write_shards

pytestmark = pytest.mark.gpu

DT = torch.bfloat16
FP8 = torch.float8_e4m3fn


def _engine(row, H, I, E, K, L=1, max_tokens=1024, **kw):
    from moe_infinity_b200 import MoEEngine
    if row:
        return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                         expert_dtype=FP8, fp8_scales="row", **kw)
    return MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, max_tokens=max_tokens,
                     pack_weights=False, **kw)


def _adversarial(q, s):
    """Every finite e4m3 code in rows 0..127, an all-zero row 200, and row scales spanning 2^-30 .. 2^10."""
    codes = torch.tensor([c for c in range(256) if c & 0x7f != 0x7f], dtype=torch.uint8, device=q.device)
    qb = q.view(torch.uint8)
    qb[:128] = codes.repeat(128 * qb.shape[1] // len(codes) + 1)[:128 * qb.shape[1]].view(128, -1)
    qb[200] = 0
    r = torch.arange(s.shape[0], device=s.device)
    s.copy_(torch.exp2(((r * 7) % 41 - 30).float()) * (1 + (r % 5).float() / 7))
    return q, s


def _row_weights(seed, H, I, E, shapes=None, adversarial=False):
    """[(q list, s list)] per expert from quantize_row of N(0, 0.02); shapes default to Mixtral's w1 | w2 | w3."""
    from moe_infinity_b200.fp8 import quantize_row
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = shapes or [(I, H), (H, I), (I, H)]
    out = []
    for e in range(E):
        qs, ss = [], []
        for m, shp in enumerate(shapes):
            q, s = quantize_row(torch.randn(*shp, generator=g, device="cuda") * 0.02)
            if adversarial and m != 2 and e % 2 == 0:
                q, s = _adversarial(q, s)
            qs.append(q)
            ss.append(s)
        out.append((qs, ss))
    return out


def _deq(ws):
    from moe_infinity_b200.fp8 import dequantize_row
    return [[dequantize_row(q, s) for q, s in zip(qs, ss)] for qs, ss in ws]


def _load_pair(a, b, ws, layer=0, resident=True):
    for e, ((qs, ss), w) in enumerate(zip(ws, _deq(ws))):
        if resident:
            a.load_expert(layer, e, qs, scales=ss)
            b.load_expert(layer, e, w)
        else:
            a.register_expert(layer, e, [q.cpu() for q in qs], scales=[s.cpu().reshape(-1, 1) for s in ss])
            b.register_expert(layer, e, [t.cpu() for t in w])


def _fwd(eng, x, layer=0, **kw):
    out = eng.forward(layer, x, **kw)
    torch.cuda.synchronize()
    return out.clone()


@pytest.mark.parametrize("adversarial", [False, True], ids=["normal_weights", "adversarial"])
def test_row_matches_bf16_mixtral_fullsize(adversarial, lib_built):
    from moe_infinity_b200.fp8 import expert_blob_bytes
    H, I, E, K = 4096, 14336, 8, 2
    ws = _row_weights(1, H, I, E, adversarial=adversarial)
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    a, b = _engine(True, H, I, E, K), _engine(False, H, I, E, K)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.set_gate(0, gate)
    assert a.stats()["slot_bytes"] == expert_blob_bytes(H, I, "row") == 3 * H * I + 4 * (2 * I + H)
    for T in (1, 8, 64, 256, 257, 1024):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        for _ in range(2):
            ya, yb, yb2 = _fwd(a, x), _fwd(b, x), _fwd(b, x)
            _equal_where_reproducible(ya, yb, yb2, f"T={T}")
        if not adversarial:
            assert torch.isfinite(ya.float()).all() and ya.float().abs().max() > 0
    a.close(); b.close()


def test_deepseek_v3_router_with_shared_expert(lib_built):
    from moe_infinity_b200 import _lib as L
    from test_gpu_fp8_experts import _check_same
    H, I, E, K, SI = 2048, 1408, 64, 6, 2816
    ws = _row_weights(6, H, I, E, shapes=[(I, H), (I, H), (H, I)])     # gate | up | down
    g = torch.Generator(device="cuda").manual_seed(60)
    shared = [(torch.randn(SI, H, generator=g, device="cuda") * 0.02).to(DT),
              (torch.randn(SI, H, generator=g, device="cuda") * 0.02).to(DT),
              (torch.randn(H, SI, generator=g, device="cuda") * 0.02).to(DT)]
    gate = torch.randn(E, H, generator=g, device="cuda") * 0.05
    bias = torch.randn(E, generator=g, device="cuda") * 0.01
    kw = dict(max_tokens=512, expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_DEEPSEEK_V3, n_group=8, topk_group=4,
              norm_topk_prob=True, routed_scaling_factor=2.5, shared_inter=SI)
    a, b = _engine(True, H, I, E, K, **kw), _engine(False, H, I, E, K, **kw)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.register_shared(0, shared)
        eng.set_gate(0, gate)
        eng.set_gate_bias(0, bias)
    for T in (1, 8, 512):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        _check_same(a, b, x, f"T={T}")
    a.close(); b.close()


def test_qwen3_moe(lib_built):
    from moe_infinity_b200 import _lib as L
    from test_gpu_fp8_experts import _check_same
    H, I, E, K = 2048, 768, 128, 8
    ws = _row_weights(7, H, I, E, shapes=[(I, H), (I, H), (H, I)])
    gate = (torch.randn(E, H, device="cuda") * 0.05).to(DT)
    kw = dict(max_tokens=512, expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_QWEN_MOE, norm_topk_prob=True)
    a, b = _engine(True, H, I, E, K, **kw), _engine(False, H, I, E, K, **kw)
    _load_pair(a, b, ws)
    for T in (1, 8, 512):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        _check_same(a, b, x, f"T={T}", router_logits=F.linear(x, gate))
    a.close(); b.close()


def test_llama4_with_shared_expert(lib_built):
    from moe_infinity_b200 import _lib as L
    from test_gpu_llama4 import _equal_or_splitk
    H, I, E, K = 2048, 4096, 16, 1
    ws = _row_weights(8, H, I, E, shapes=[(I, H), (I, H), (H, I)])
    g = torch.Generator(device="cuda").manual_seed(80)
    shared = [(torch.randn(I, H, generator=g, device="cuda") * 0.02).to(DT),
              (torch.randn(I, H, generator=g, device="cuda") * 0.02).to(DT),
              (torch.randn(H, I, generator=g, device="cuda") * 0.02).to(DT)]
    gate = (torch.randn(E, H, generator=g, device="cuda") * 0.1).to(DT)
    kw = dict(expert_type=L.EXPERT_DEEPSEEK, router=L.ROUTER_LLAMA4, shared_inter=I)
    a, b = _engine(True, H, I, E, K, **kw), _engine(False, H, I, E, K, **kw)
    _load_pair(a, b, ws)
    for eng in (a, b):
        eng.register_shared(0, shared)
        eng.set_gate(0, gate)
    for T in (1, 16, 200, 1024):
        x = torch.randn(T, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).to(DT)
        lg = F.linear(x, gate)
        _equal_or_splitk(_fwd(a, x, router_logits=lg), _fwd(b, x, router_logits=lg), f"T={T}", a, b, T)
    a.close(); b.close()


def test_offload_and_decode_graph(lib_built):
    from moe_infinity_b200 import DecodeSession
    from test_gpu_fp8_experts import _check_same
    H, I, E, T = 1024, 2048, 8, 8
    ws = [_row_weights(10 + l, H, I, E) for l in range(2)]
    # host-backed experts ([out, 1] scales), 3 slots for 2 layers x 8 experts: every layer call evicts and re-stages
    a = _engine(True, H, I, E, 2, L=2, num_slots=3, max_tokens=64)
    b = _engine(False, H, I, E, 2, L=2, num_slots=3, max_tokens=64)
    for l in range(2):
        _load_pair(a, b, ws[l], layer=l, resident=False)
    logits = torch.randn(16, E, device="cuda").to(DT)
    for step in range(2):
        for l in range(2):
            xl = torch.randn(16, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(10 * step + l)).to(DT)
            _check_same(a, b, xl, f"step {step} layer {l}", l, router_logits=logits)
    sa = a.stats()
    assert sa["misses"] > 6 and sa["evictions"] > 0 and sa["h2d_bytes"] == sa["misses"] * a.expert_bytes
    a.close(); b.close()
    # a captured decode step replays the eager forwards of a resident row-format engine
    a = _engine(True, H, I, E, 2, L=2, max_tokens=64)
    for l in range(2):
        for e, (qs, ss) in enumerate(ws[l]):
            a.load_expert(l, e, qs, scales=ss)
        a.set_gate(l, (torch.randn(E, H, device="cuda") * 0.05).to(DT))
    sess = DecodeSession(a, T)
    sess.x_host.copy_(torch.randn(2, T, H).to(DT))
    eager = torch.stack([_fwd(a, sess.x_host[l].cuda(), l) for l in range(2)]).cpu()
    sess.capture()
    assert torch.equal(sess.step().clone(), eager)
    a.close()


# ---------------------------------------------------------------- every fp8 launch plan, exact against float64
ROW_CASES = [c for c in X.CASES if c.fmt == "fp8"]


def _row_expert(c: X.Case, seed: int) -> X.Expert:
    """Codes in {0, +-1} (gate {0, 1}) with a 2^j scale per row: gate and up j in {0, 1}, down j in {-1, 0} -- the values the
    block-format rows reach, so X.reference's budget holds."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ws, load, scales = [], [], []
    for role, (rows, cols) in X.matrix_shapes(c.etype, c.H, c.I):
        d = X._pattern(role, rows, cols, True, g, "cuda")
        lo, hi = (-1, 0) if role == "down" else (0, 1)
        s = torch.pow(2.0, torch.randint(lo, hi + 1, (rows,), generator=g, device="cuda").double())
        ws.append((d * s[:, None]).to(DT))
        load.append(d.float().to(FP8))
        scales.append(s.float())
    return X.Expert(ws, load, scales)


_cur = {"key": None}


def _engine_for(c: X.Case):
    if _cur["key"] == c.engine_key:
        return _cur
    if _cur.get("eng") is not None:
        _cur["eng"].close()
    _cur.clear()
    _cur["key"] = None
    torch.cuda.empty_cache()
    from moe_infinity_b200 import _lib as L
    max_t = max(r.T for r in ROW_CASES if r.engine_key == c.engine_key)
    eng = _engine(True, c.H, c.I, c.E, c.k, max_tokens=max(max_t, 16), expert_type=X.ETYPE[c.etype], router=L.ROUTER_MIXTRAL)
    experts = [_row_expert(c, 1000 + e) for e in range(c.E)]
    for e, ex in enumerate(experts):
        eng.load_expert(0, e, ex.load, scales=ex.scales)
    torch.cuda.synchronize()
    _cur.update(key=c.engine_key, eng=eng, experts=experts)
    return _cur


@pytest.mark.parametrize("name", [c.name for c in ROW_CASES])
def test_row_expert_gemms_are_exact(lib_built, name):
    from test_gpu_gemm_exact import _replay_combine, _route_and_run, _same
    c = X.BY_NAME[name]
    st = _engine_for(c)
    eng, experts = st["eng"], st["experts"]
    T, k = c.T, c.k
    x = X.make_x(T, c.H, DT, seed=T, dev="cuda")
    out = _route_and_run(c, eng, x)
    torch.cuda.synchronize()
    assert eng.ws("counts", T).tolist() == list(c.counts), "routing did not produce the designed counts"
    offs = eng.ws("offsets", T).tolist()
    perm = eng.ws("perm_token", T).long()
    hmid, y = eng.ws("hmid", T), eng.ws("y", T)
    y_all = torch.empty(T * k, c.H, dtype=torch.float32, device="cuda")
    for e in range(c.E):
        r0, r1 = offs[e], offs[e + 1]
        if r0 == r1:
            continue
        h_ref, y_ref = X.reference(c, x[perm[r0:r1]], experts[e].w)
        _same(hmid[r0:r1], h_ref, f"{name} expert {e} hmid")
        _same(y[r0:r1], y_ref, f"{name} expert {e} y")
        y_all[r0:r1] = y_ref
    _same(out.reshape(T, c.H), _replay_combine(c, eng, y_all, None), f"{name} layer output")
    # the down projection alone, on dense small integers
    h2 = X.make_hmid(T * k, c.I, DT, seed=7 + T, dev="cuda")
    hmid.copy_(h2)
    y.zero_()
    eng.run_experts(0, T, phases=2)
    torch.cuda.synchronize()
    for e in range(c.E):
        r0, r1 = offs[e], offs[e + 1]
        if r0 < r1:
            _same(y[r0:r1], X.reference(c, None, experts[e].w, hmid=h2[r0:r1])[1], f"{name} expert {e} y (dense hmid)")


def test_release_exact_engine(lib_built):
    if _cur.get("eng") is not None:
        _cur["eng"].close()
    _cur.clear()
    _cur["key"] = None
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- checkpoint loaders end to end
def _equal_or_atomics(got, want, what):
    """torch.equal, or -- fp32 atomics of a down projection split over three or more CTAs add in arrival order, so two runs
    of one engine may differ in the last bits -- within test_gpu_parity.hidden_close's bound."""
    from test_gpu_parity import hidden_close
    if not torch.equal(got, want):
        hidden_close(got.reshape(-1, got.shape[-1]), want.reshape(-1, want.shape[-1]).cpu(), None, DT, what)


def _equal_where_reproducible(got, want, want_again, what):
    """torch.equal whenever the reference engine reproduces its own output, else _equal_or_atomics."""
    if torch.equal(want, want_again):
        assert torch.equal(got, want), f"{what}: {(got.float() - want.float()).abs().max().item()}"
    _equal_or_atomics(got, want, what)


def test_llama4_fp8_checkpoint_into_patched_model(lib_built, tmp_path):
    tr = pytest.importorskip("transformers")
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200.fp8 import dequantize_row, quantize_row
    from moe_infinity_b200.hf import load_fp8_checkpoint, patch_llama4
    cfg = tr.Llama4TextConfig(vocab_size=512, hidden_size=256, intermediate_size=256, intermediate_size_mlp=512,
                              num_hidden_layers=4, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                              num_local_experts=16, num_experts_per_tok=1, interleave_moe_layer_step=2,
                              max_position_embeddings=128)
    torch.manual_seed(0)
    model = tr.Llama4ForCausalLM(cfg).to(DT).cuda().eval()
    H, I, E = cfg.hidden_size, cfg.intermediate_size, cfg.num_local_experts
    tensors = {}
    with torch.no_grad():
        for l, layer in enumerate(model.model.layers):
            ff = layer.feed_forward
            if not hasattr(ff, "router"):
                continue
            ff.router.weight.mul_(20.0)
            b = f"model.layers.{l}.feed_forward"
            # fbgemm layout: gate_up_proj [E, H, 2I] with a scale per output column, down_proj [E, I, H] per output column
            gu, gus, dn, dns = [], [], [], []
            for e in range(E):
                q, s = quantize_row(torch.randn(2 * I, H, device="cuda") * 0.02)        # [2I, H]: row j = output j
                gu.append(q.view(torch.uint8).t().contiguous().view(FP8))
                gus.append(s.reshape(1, 2 * I))
                ff.experts.gate_up_proj[e].copy_(dequantize_row(q, s).t())
                q, s = quantize_row(torch.randn(H, I, device="cuda") * 0.02)
                dn.append(q.view(torch.uint8).t().contiguous().view(FP8))
                dns.append(s.reshape(H, 1))
                ff.experts.down_proj[e].copy_(dequantize_row(q, s).t())
            tensors.update({f"{b}.experts.gate_up_proj": torch.stack(gu).cpu(), f"{b}.experts.gate_up_proj_scale": torch.stack(gus).cpu(),
                            f"{b}.experts.down_proj": torch.stack(dn).cpu(), f"{b}.experts.down_proj_scale": torch.stack(dns).cpu(),
                            f"{b}.router.weight": ff.router.weight.cpu()})
            for n in ("gate_proj", "up_proj", "down_proj"):          # an FbgemmFp8Linear shared expert
                w = getattr(ff.shared_expert, n).weight
                q, s = quantize_row(w)
                w.copy_(dequantize_row(q, s))
                tensors[f"{b}.shared_expert.{n}.weight"] = q.cpu()
                tensors[f"{b}.shared_expert.{n}.weight_scale"] = s.reshape(-1, 1).cpu()
    paths = write_shards(str(tmp_path), tensors)
    ref = copy.deepcopy(model)            # bf16 experts = the dequantised checkpoint
    patch_llama4(ref, max_tokens=256)
    ours = copy.deepcopy(model)
    from moe_infinity_b200 import MoEEngine
    eng = MoEEngine(num_layers=4, num_experts=E, hidden=H, inter=I, top_k=1, dtype=DT, expert_type=L.EXPERT_DEEPSEEK,
                    router=L.ROUTER_LLAMA4, shared_inter=I, max_tokens=256, expert_dtype=FP8, fp8_scales="row")
    patch_llama4(ours, engine=eng)
    # the checkpoint's codes and scales replace what patch_llama4 quantised from the model
    assert load_fp8_checkpoint(eng, paths, {"quant_method": "fbgemm_fp8", "modules_to_not_convert": []}, "llama4") == [1, 3]
    ids = torch.randint(0, 512, (2, 24), device="cuda")
    with torch.no_grad():
        a, b = ref(ids).logits, ours(ids).logits
    _equal_or_atomics(b, a, "llama4 logits")


@pytest.mark.parametrize("model_type", ["qwen3_moe", "deepseek_v3"])
def test_block_fp8_checkpoint_equals_hand_fed_engine(lib_built, tmp_path, model_type):
    from moe_infinity_b200 import MoEEngine
    from moe_infinity_b200 import _lib as L
    from moe_infinity_b200.fp8 import quantize_block128
    from moe_infinity_b200.hf import load_fp8_checkpoint
    H, I, E, K, SI, Lyr = 512, 256, 16, 4, 512, 2
    v3 = model_type == "deepseek_v3"
    kw = dict(num_layers=Lyr, num_experts=E, hidden=H, inter=I, top_k=K, dtype=DT, expert_type=L.EXPERT_DEEPSEEK,
              max_tokens=256, expert_dtype=FP8, norm_topk_prob=True)
    kw.update(dict(router=L.ROUTER_DEEPSEEK_V3, shared_inter=SI, n_group=4, topk_group=2, routed_scaling_factor=2.5,
                   gate_dtype=torch.float32) if v3 else dict(router=L.ROUTER_QWEN_MOE))
    g = torch.Generator().manual_seed(5)
    t, by_hand = {}, []
    for l in range(Lyr):
        b = f"model.layers.{l}.mlp"
        mats = []
        for e in range(E):
            qs, ss = [], []
            for n, shp in (("gate_proj", (I, H)), ("up_proj", (I, H)), ("down_proj", (H, I))):
                q, s = quantize_block128(torch.randn(*shp, generator=g) * 0.02)
                t[f"{b}.experts.{e}.{n}.weight"], t[f"{b}.experts.{e}.{n}.weight_scale_inv"] = q, s
                qs.append(q)
                ss.append(s)
            mats.append((qs, ss))
        gate = torch.randn(E, H, generator=g) * 0.05
        t[f"{b}.gate.weight"] = gate if v3 else gate.to(DT)
        shared = None
        if v3:
            t[f"{b}.gate.e_score_correction_bias"] = torch.randn(E, generator=g) * 0.01
            shared = [(torch.randn(*shp, generator=g) * 0.02).to(DT) for shp in ((SI, H), (SI, H), (H, SI))]
            for n, w in zip(("gate_proj", "up_proj", "down_proj"), shared):
                t[f"{b}.shared_experts.{n}.weight"] = w
        by_hand.append((mats, t[f"{b}.gate.weight"], t.get(f"{b}.gate.e_score_correction_bias"), shared))
    paths = write_shards(str(tmp_path), t)
    a, h = MoEEngine(**kw), MoEEngine(**kw)
    qc = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}
    assert load_fp8_checkpoint(a, paths, qc, model_type) == list(range(Lyr))
    for l, (mats, gate, bias, shared) in enumerate(by_hand):
        for e, (qs, ss) in enumerate(mats):
            h.load_expert(l, e, qs, scales=ss)
        h.set_gate(l, gate)
        if v3:
            h.set_gate_bias(l, bias)
            h.register_shared(l, shared)
    for T in (1, 8, 200):
        x = torch.randn(T, H, generator=torch.Generator().manual_seed(T)).to(DT).cuda()
        for l in range(Lyr):
            kwf = {} if v3 else dict(router_logits=F.linear(x, by_hand[l][1].cuda()))
            oa = _fwd(a, x, l, **kwf)
            ha = a.ws("hmid", T).clone()
            oh = _fwd(h, x, l, **kwf)
            # the gate/up GEMM has no split-K: its outputs must agree bit for bit
            assert torch.equal(ha, h.ws("hmid", T)), f"{model_type} T={T} layer {l}: gate/up outputs differ"
            _equal_or_atomics(oa, oh, f"{model_type} T={T} layer {l}")
    a.close(); h.close()
