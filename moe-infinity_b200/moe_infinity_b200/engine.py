"""MoEEngine: thin Python host object over the C-ABI context (include/b2m.h).

Plays the role of the reference's two pybind objects -- `prefetch_handle` (weight residency,
prefetch, cache) and `expert_dispatcher` (expert execution) -- for the MoE block hot path
(core/python/py_archer_prefetch.cpp:10-92), plus the fused fast path `forward`.
PyTorch is used for device memory and streams only; all math runs in libb2m.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib as L
from . import fp8 as F8
from . import int4 as I4

_TORCH2INT = {torch.bfloat16: L.DTYPE_BF16, torch.float32: L.DTYPE_F32, torch.float16: L.DTYPE_F16}
_INT2TORCH = {v: k for k, v in _TORCH2INT.items()}


class _DevArray:
    """Zero-copy view of a raw device pointer through __cuda_array_interface__."""

    def __init__(self, ptr: int, shape: Tuple[int, ...], typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


def _view(ptr: int, shape: Tuple[int, ...], dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    if dtype in (torch.bfloat16, torch.float16):
        t = torch.as_tensor(_DevArray(ptr, shape, "<i2"), device=device)
        return t.view(dtype)
    typestr = {torch.float32: "<f4", torch.int32: "<i4", torch.uint8: "|u1"}[dtype]
    return torch.as_tensor(_DevArray(ptr, shape, typestr), device=device)


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


# routers whose logits are an nn.Linear of the model: gate weight and logits in the model dtype
_MODEL_DTYPE_ROUTERS = (L.ROUTER_MIXTRAL, L.ROUTER_QWEN_MOE, L.ROUTER_LLAMA4)

class MoEEngine:
    def __init__(self, *, num_layers: int, num_experts: int, hidden: int, inter: int, top_k: int,
                 dtype: torch.dtype = torch.bfloat16, expert_type: int = L.EXPERT_MIXTRAL,
                 router: int = L.ROUTER_MIXTRAL, numerics: int = L.NUMERICS_REFERENCE, max_tokens: int = 256,
                 num_slots: int = 0, device_memory_ratio: float = 0.0, shared_inter: int = 0, n_group: int = 1,
                 topk_group: int = 1, norm_topk_prob: bool = False, routed_scaling_factor: float = 1.0,
                 expert_capacity: int = 0, gate_dtype: Optional[torch.dtype] = None, device: int = 0,
                 max_inflight_prefetch: int = 2, h2d_chunk_bytes: int = 0, gemm_impl: int = 0,
                 cache_policy: int = L.CACHE_REFERENCE, lookahead_prefetch: bool = False, freq_alpha: float = 0.0,
                 pack_weights: bool = True, expert_dtype: Optional[torch.dtype] = None, fp8_scales: str = "block128"):
        """expert_dtype: None = the routed experts are stored in `dtype`; torch.float8_e4m3fn = FP8 E4M3 with one fp32 scale
        per 128x128 block (`fp8.py`; `dtype` stays the activation dtype and must be bf16; register_expert / load_expert then
        take the three e4m3 matrices and their scale grids); torch.uint4 = 4-bit codes with a 16-bit scale and a 4-bit zero
        point per 128 inputs (`int4.py`; register_expert / load_expert then take the three packed code matrices with scales=
        and zeros=).  The scales are of `dtype`: bf16 (B2M_WEIGHTS_INT4_G128) or float16 (B2M_WEIGHTS_INT4_G128_F16, the
        AWQ / GPTQ format: `int4.from_awq`, `int4.from_gptq`, `hf.load_int4_checkpoint`).
        fp8_scales (fp8 engines): "block128" (the default, above) or "row": one fp32 scale per output channel
        (B2M_WEIGHTS_FP8_E4M3_ROW, `fp8.dequantize_row`; the fbgemm FP8 format, `hf.load_fp8_checkpoint`); the scales
        given to register_expert / load_expert are then float32 [out] (or [out, 1]) vectors."""
        self.lib = L.load()
        if not torch.cuda.is_available():
            raise RuntimeError("moe_infinity_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        if dtype not in _TORCH2INT:
            raise ValueError(f"unsupported dtype {dtype}")
        if expert_dtype is not None and expert_dtype not in (torch.float8_e4m3fn, torch.uint4):
            raise ValueError(f"unsupported expert_dtype {expert_dtype} (None, torch.float8_e4m3fn or torch.uint4)")
        self.fp8 = expert_dtype == torch.float8_e4m3fn
        if fp8_scales not in ("block128", "row"):
            raise ValueError(f"fp8_scales {fp8_scales!r}: 'block128' or 'row'")
        if fp8_scales != "block128" and not self.fp8:
            raise ValueError("fp8_scales goes with an fp8 engine (expert_dtype=torch.float8_e4m3fn)")
        self.fp8_scales = fp8_scales if self.fp8 else None
        self.int4 = expert_dtype == torch.uint4
        if self.fp8 and dtype != torch.bfloat16:
            raise ValueError("fp8 experts compute with bf16 activations: dtype must be torch.bfloat16")
        if self.int4 and dtype not in (torch.bfloat16, torch.float16):
            raise ValueError("int4 experts compute with 16-bit activations: dtype must be torch.bfloat16 or torch.float16")
        self.dtype = dtype
        self.device = torch.device("cuda", device)
        self.L, self.E, self.H, self.I, self.k = num_layers, num_experts, hidden, inter, top_k
        self.shared_inter = shared_inter
        self.expert_type = expert_type
        self.router = router
        # Mixtral, Qwen and Llama 4 routers are nn.Linear layers of the model: their weight is in the model dtype
        gate_dtype = gate_dtype or (dtype if router in _MODEL_DTYPE_ROUTERS else torch.float32)
        self.gate_dtype = gate_dtype
        cfg = L.Config()
        cfg.struct_size = C.sizeof(L.Config)
        cfg.device = device
        cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k = num_layers, num_experts, hidden, inter, top_k
        cfg.dtype = _TORCH2INT[dtype]
        cfg.expert_type, cfg.router, cfg.numerics = expert_type, router, numerics
        cfg.max_tokens, cfg.num_slots, cfg.shared_inter = max_tokens, num_slots, shared_inter
        cfg.n_group, cfg.topk_group, cfg.norm_topk_prob = n_group, topk_group, int(bool(norm_topk_prob))
        cfg.expert_capacity = expert_capacity
        cfg.routed_scaling_factor = routed_scaling_factor
        cfg.gate_dtype = _TORCH2INT[gate_dtype]
        cfg.device_memory_ratio = device_memory_ratio
        cfg.max_inflight_prefetch = max_inflight_prefetch
        cfg.h2d_chunk_bytes = h2d_chunk_bytes
        # gemm_impl 2: tensor cores without the packed copy of the experts (see include/b2m.h)
        cfg.gemm_impl = 2 if (gemm_impl == 0 and not pack_weights) else gemm_impl
        cfg.cache_policy = cache_policy
        cfg.lookahead_prefetch = int(lookahead_prefetch)
        cfg.freq_alpha = freq_alpha
        self.cfg = cfg
        self.max_tokens = max_tokens
        h = C.c_void_p()
        torch.cuda.set_device(self.device)
        fmt = L.WEIGHTS_MODEL_DTYPE
        if self.fp8:
            fmt = L.WEIGHTS_FP8_E4M3_ROW if fp8_scales == "row" else L.WEIGHTS_FP8_E4M3_B128
        elif self.int4:
            fmt = L.WEIGHTS_INT4_G128_F16 if dtype == torch.float16 else L.WEIGHTS_INT4_G128
        L.check(None, self.lib.b2m_ctx_create_ex(C.byref(cfg), fmt, C.byref(h)))
        self._h = h
        self._blobs: Dict[Tuple[int, int], torch.Tensor] = {}
        self._gates: Dict[int, torch.Tensor] = {}
        self._biases: Dict[int, torch.Tensor] = {}
        self._perms: Dict[int, torch.Tensor] = {}
        self._shared_gates: Dict[int, torch.Tensor] = {}
        es = self.esize = 4 if dtype == torch.float32 else 2   # fp32 experts (dtype int 1) run on the CUDA-core fp32 path
        self.expert_bytes = self.stats()["slot_bytes"]          # one expert blob in the context's weight format
        self.shared_bytes = 3 * hidden * shared_inter * es

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if getattr(self, "_h", None):
            self.lib.b2m_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, code):
        return L.check(self._h, code)

    # ------------------------------------------------------------------ weights
    def _pack(self, tensors: Sequence[torch.Tensor], nbytes: int, pin: bool) -> torch.Tensor:
        """Concatenate tensors in the reference's tensor_ids order into one host blob
        (core/model/model_topology.cpp:429-431)."""
        blob = torch.empty(nbytes, dtype=torch.uint8, pin_memory=pin)
        off = 0
        for t in tensors:
            t = t.detach().to("cpu", self.dtype).contiguous()
            n = t.numel() * self.esize
            blob[off:off + n] = t.view(torch.uint8).reshape(-1)
            off += n
        if off != nbytes:
            raise ValueError(f"expert tensors total {off} bytes, expected {nbytes}")
        return blob

    def _fp8_parts(self, tensors: Sequence[torch.Tensor], scales: Optional[Sequence[torch.Tensor]]) -> List[torch.Tensor]:
        """The fp8 expert blob's parts as flat uint8 tensors: three e4m3 matrices, then their fp32 scale grids (row scales:
        vectors)."""
        if scales is None:
            raise ValueError("an fp8 engine needs the three scale grids: scales=(s1, s2, s3)")
        if len(tensors) != 3 or len(scales) != 3:
            raise ValueError("an fp8 expert is three e4m3 matrices and three scale grids")
        H, I = self.H, self.I
        # nn.Linear [out, in]: Mixtral w1 | w2 | w3 = gate, down, up; DeepSeek gate | up | down
        shapes = [(I, H), (H, I), (I, H)] if self.expert_type == L.EXPERT_MIXTRAL else [(I, H), (I, H), (H, I)]
        parts = []
        for t, shp in zip(tensors, shapes):
            if t.dtype != torch.float8_e4m3fn or tuple(t.shape) != shp:
                raise ValueError(f"expected a float8_e4m3fn {shp} matrix, got {t.dtype} {tuple(t.shape)}")
            parts.append(t.detach().contiguous().view(torch.uint8).reshape(-1))
        for s, shp in zip(scales, shapes):
            if self.fp8_scales == "row":
                if s.dtype != torch.float32 or tuple(s.shape) not in ((shp[0],), (shp[0], 1)):
                    raise ValueError(f"expected a float32 ({shp[0]},) or ({shp[0]}, 1) row-scale vector, got {s.dtype} "
                                     f"{tuple(s.shape)}")
                parts.append(s.detach().contiguous().view(torch.uint8).reshape(-1))
                continue
            want = (shp[0] // F8.BLOCK, shp[1] // F8.BLOCK)
            if s.dtype != torch.float32 or tuple(s.shape) != want:
                raise ValueError(f"expected a float32 {want} scale grid, got {s.dtype} {tuple(s.shape)}")
            parts.append(s.detach().contiguous().view(torch.uint8).reshape(-1))
        return parts

    def _int4_parts(self, tensors: Sequence[torch.Tensor], scales: Optional[Sequence[torch.Tensor]],
                    zeros: Optional[Sequence[torch.Tensor]]) -> List[torch.Tensor]:
        """The int4 expert blob's parts as flat uint8 tensors: three packed code matrices, then their tile-major group
        grids (int4.py)."""
        if scales is None or zeros is None:
            raise ValueError("an int4 engine needs the three scale and zero-point grids: scales=(s1, s2, s3), zeros=(z1, z2, z3)")
        if len(tensors) != 3 or len(scales) != 3 or len(zeros) != 3:
            raise ValueError("an int4 expert is three code matrices, three scale grids and three zero-point grids")
        H, I = self.H, self.I
        # nn.Linear [out, in]: Mixtral w1 | w2 | w3 = gate, down, up; DeepSeek gate | up | down
        shapes = [(I, H), (H, I), (I, H)] if self.expert_type == L.EXPERT_MIXTRAL else [(I, H), (I, H), (H, I)]
        parts, grids = [], []
        for t, s, z, (r, c) in zip(tensors, scales, zeros, shapes):
            if t.dtype != torch.uint8 or tuple(t.shape) != (r, c // 2):
                raise ValueError(f"expected a uint8 {(r, c // 2)} code matrix (two codes per byte), got {t.dtype} {tuple(t.shape)}")
            want = (r, c // I4.GROUP)
            if s.dtype != self.dtype or tuple(s.shape) != want:   # (the scales are of the activations' type: no rounding)
                raise ValueError(f"expected a {self.dtype} {want} scale grid, got {s.dtype} {tuple(s.shape)}")
            if z.dtype != torch.uint8 or tuple(z.shape) != want:
                raise ValueError(f"expected a uint8 {want} zero-point grid, got {z.dtype} {tuple(z.shape)}")
            parts.append(t.detach().contiguous().reshape(-1))
            grids.append(I4.pack_groups(s.detach(), z.detach().to(s.device)))
        return parts + grids

    def _quant_parts(self, tensors, scales, zeros) -> Optional[List[torch.Tensor]]:
        """The blob parts of a quantised engine's expert; None on a model-dtype engine (which takes no scales / zeros)."""
        if self.fp8:
            if zeros is not None:
                raise ValueError("zeros go with the int4 codes of an int4 engine (expert_dtype=torch.uint4)")
            return self._fp8_parts(tensors, scales)
        if self.int4:
            return self._int4_parts(tensors, scales, zeros)
        if scales is not None or zeros is not None:
            raise ValueError("scales / zeros are only taken by an fp8 or int4 engine (expert_dtype=torch.float8_e4m3fn / torch.uint4)")
        return None

    def register_expert(self, layer: int, expert: int, tensors: Sequence[torch.Tensor], pin: bool = True,
                        scales: Optional[Sequence[torch.Tensor]] = None, zeros: Optional[Sequence[torch.Tensor]] = None):
        """Host-backed expert (can be staged in and evicted).  tensors: Mixtral (w1,w2,w3),
        DeepSeek (gate,up,down), Switch (wi,wo), NLLB/FSGPT (fc1,fc1_bias,fc2,fc2_bias) -- nn.Linear [out,in] layout.
        fp8 engine: the three float8_e4m3fn matrices and `scales`, their float32 [out/128, in/128] grids (fp8_scales="row":
        float32 [out] vectors).
        int4 engine: the three uint8 [out, in/2] code matrices (int4.quantize_g128), `scales` ([out, in/128] of the engine's
        dtype, bfloat16 or float16) and `zeros` (uint8 [out, in/128])."""
        parts = self._quant_parts(tensors, scales, zeros)
        if parts is not None:
            blob = torch.zeros(self.expert_bytes, dtype=torch.uint8, pin_memory=pin)
            off = 0
            for part in parts:
                blob[off:off + part.numel()] = part.cpu()
                off += part.numel()
        else:
            blob = self._pack(tensors, self.expert_bytes, pin)
        self._blobs[(layer, expert)] = blob
        self._ck(self.lib.b2m_register_expert(self._h, layer, expert, C.c_void_p(blob.data_ptr()), blob.numel()))

    def register_expert_on_store(self, layer: int, expert: int, reader, tensor_ids: Sequence[int]):
        """Disk-backed expert (SURVEY §8f N3): its weights stay on the reference-format store behind `reader`
        (`store.NativeStoreReader`); a miss streams them disk -> pinned staging ring -> HBM slot in chunks.  `tensor_ids` in
        blob order (what the reference's `register_expert` receives, model_offload.py:851-853)."""
        ids = (C.c_uint32 * len(tensor_ids))(*[int(t) for t in tensor_ids])
        self._stores = getattr(self, "_stores", [])
        self._stores.append(reader)                                    # the store must outlive the context
        self._blobs.pop((layer, expert), None)
        self._ck(self.lib.b2m_register_expert_on_store(self._h, layer, expert, reader.handle, ids, len(tensor_ids)))

    def make_resident(self, layer: int, expert: int, pin: bool = False):
        self._ck(self.lib.b2m_make_resident(self._h, layer, expert, 1 if pin else 0, C.c_void_p(_stream_ptr())))

    def expert_device_view(self, layer: int, expert: int) -> Optional[torch.Tensor]:
        p = C.c_void_p()
        self._ck(self.lib.b2m_expert_dev_ptr(self._h, layer, expert, C.byref(p)))
        if not p.value:
            return None
        if self.fp8 or self.int4:   # the fp8 / int4 expert blob (fp8.py / int4.py): quantised matrices, then their grids
            return _view(p.value, (self.expert_bytes,), torch.uint8, self.device)
        return _view(p.value, (self.expert_bytes // self.esize,), self.dtype, self.device)

    def load_expert(self, layer: int, expert: int, tensors: Optional[Sequence[torch.Tensor]] = None,
                    scales: Optional[Sequence[torch.Tensor]] = None, zeros: Optional[Sequence[torch.Tensor]] = None):
        """HBM-only expert: claims a slot, pins it, fills it from `tensors` (any device) if given.
        Returns the flat device view of the slot so callers can initialise it in place.  Writes through the view must be
        issued (on the current stream) before the next forward of this layer; the second eager forward after the load packs
        the slot for the decode GEMMs (pack_weights=True); to change the weights later, call load_expert again and write through the view it returns.
        fp8 engine: `tensors` are the three float8_e4m3fn matrices and `scales` their float32 grids; the view is uint8.
        int4 engine: `tensors` are the three uint8 code matrices, `scales` / `zeros` their grids (the engine's dtype / uint8);
        the view is uint8."""
        parts = None
        if tensors is not None:
            parts = self._quant_parts(tensors, scales, zeros)
        elif scales is not None or zeros is not None:
            raise ValueError("scales / zeros go with the quantised matrices of an fp8 or int4 engine")
        self._ck(self.lib.b2m_make_resident(self._h, layer, expert, 1 | 2, C.c_void_p(_stream_ptr())))
        v = self.expert_device_view(layer, expert)
        if parts is not None:
            off = 0
            for part in parts:
                v[off:off + part.numel()].copy_(part)
                off += part.numel()
            v[off:].zero_()
        elif tensors is not None:
            off = 0
            for t in tensors:
                n = t.numel()
                v[off:off + n].copy_(t.detach().reshape(-1).to(self.dtype))
                off += n
            if off != v.numel():
                raise ValueError("expert tensors do not fill the slot")
        return v

    def register_shared(self, layer: int, tensors: Sequence[torch.Tensor]):
        blob = self._pack(tensors, self.shared_bytes, False)
        self._ck(self.lib.b2m_register_shared(self._h, layer, C.c_void_p(blob.data_ptr()), blob.numel()))

    def set_gate(self, layer: int, weight: torch.Tensor):
        w = weight.detach().to(self.device, self.gate_dtype).contiguous()
        self._gates[layer] = w
        self._ck(self.lib.b2m_set_gate(self._h, layer, C.c_void_p(w.data_ptr())))

    def set_gate_bias(self, layer: int, bias: torch.Tensor):
        """DeepSeek-V3 router (ROUTER_DEEPSEEK_V3): the layer's e_score_correction_bias [E].  fp32, or bf16 (upcast exactly;
        a block cast with .to(bf16) holds it in bf16)."""
        if self.router != L.ROUTER_DEEPSEEK_V3:
            raise ValueError("set_gate_bias needs a DeepSeek-V3 engine (router=ROUTER_DEEPSEEK_V3)")
        if bias.dtype not in (torch.float32, torch.bfloat16) or tuple(bias.shape) != (self.E,):
            raise ValueError(f"expected a float32 or bfloat16 [{self.E}] bias, got {bias.dtype} {tuple(bias.shape)}")
        b = bias.detach().to(self.device, torch.float32).contiguous()
        self._biases[layer] = b                # borrowed by the context: keep it alive
        self._ck(self.lib.b2m_set_gate_bias(self._h, layer, C.c_void_p(b.data_ptr())))

    def set_shared_gate(self, layer: int, weight: torch.Tensor):
        """Qwen2-MoE (router=ROUTER_QWEN_MOE with shared_inter > 0): the layer's shared_expert_gate.weight, [1, H] or [H] in
        the model dtype.  The combine scales the shared expert's output by sigmoid(x . weight), every op in the model dtype."""
        if self.router != L.ROUTER_QWEN_MOE or self.shared_inter <= 0:
            raise ValueError("set_shared_gate needs a Qwen-MoE engine with shared experts (router=ROUTER_QWEN_MOE, shared_inter > 0)")
        if weight.dtype != self.dtype or tuple(weight.shape) not in ((1, self.H), (self.H,)):
            raise ValueError(f"expected a {self.dtype} [1, {self.H}] or [{self.H}] shared-expert gate, got {weight.dtype} "
                             f"{tuple(weight.shape)}")
        w = weight.detach().reshape(self.H).to(self.device).contiguous()
        self._shared_gates[layer] = w          # borrowed by the context: keep it alive
        self._ck(self.lib.b2m_set_shared_gate(self._h, layer, C.c_void_p(w.data_ptr())))

    def set_input_perm(self, layer: int, perm: Optional[torch.Tensor]):
        """Act-order GPTQ on an f16 int4 engine (B2M_WEIGHTS_INT4_G128_F16): perm int [E, H], row e a permutation of
        0..H-1 (`int4.from_gptq_act_order`); the routing kernels gather column j of expert e's rows from x[t][perm[e][j]],
        so expert e's gate/up matrices are loaded as W[:, perm[e]].  None returns the layer to natural order.  The
        workspace rows "xp" and "hmid" of such a layer hold permuted activations."""
        if perm is None:
            self._ck(self.lib.b2m_set_input_perm(self._h, layer, None))
            self._perms.pop(layer, None)
            return
        if perm.dtype not in (torch.int16, torch.int32, torch.int64, torch.uint16) or tuple(perm.shape) != (self.E, self.H):
            raise ValueError(f"expected an integer [{self.E}, {self.H}] permutation table, got {perm.dtype} {tuple(perm.shape)}")
        p = perm.detach().to(torch.int64)
        if self.H > 65536 or not torch.equal(p.sort(dim=1).values.cpu(), torch.arange(self.H).expand(self.E, self.H)):
            raise ValueError("every row of the input permutation must be a permutation of 0..H-1")
        t = p.to(torch.int32).to(torch.uint16).to(self.device).contiguous()
        self._ck(self.lib.b2m_set_input_perm(self._h, layer, C.c_void_p(t.data_ptr())))
        self._perms[layer] = t                 # borrowed by the context: keep it alive

    # ------------------------------------------------------------------ hot path
    def _router_args(self, router_logits, scores):
        if scores is not None:
            s = scores.to(self.device, torch.float32).contiguous()
            return s, 2, L.DTYPE_F32
        if router_logits is not None:
            r = router_logits.to(self.device).contiguous()
            return r, 1, _TORCH2INT[r.dtype]
        return None, 0, 0

    def _check_x(self, x: torch.Tensor) -> torch.Tensor:
        if x.device != self.device or x.dtype != self.dtype:
            raise ValueError(f"x must be {self.dtype} on {self.device}")
        x2 = x.reshape(-1, self.H)
        return x2 if x2.is_contiguous() else x2.contiguous()

    def forward(self, layer: int, x: torch.Tensor, router_logits: Optional[torch.Tensor] = None,
                scores: Optional[torch.Tensor] = None, seq_len: int = 0, out: Optional[torch.Tensor] = None):
        """out[T,H] = MoE(layer)(x[T,H]).  One asynchronous call on the current stream."""
        x2 = self._check_x(x)
        T = x2.shape[0]
        if out is None:
            out = torch.empty_like(x2)
        rin, kind, rdt = self._router_args(router_logits, scores)
        self._ck(self.lib.b2m_moe_forward(self._h, layer, C.c_void_p(x2.data_ptr()),
                                          C.c_void_p(rin.data_ptr() if rin is not None else 0), kind, rdt, T, seq_len,
                                          C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr())))
        return out.view(x.shape)

    def route(self, layer: int, x: torch.Tensor, router_logits=None, scores=None, seq_len: int = 0):
        x2 = self._check_x(x)
        rin, kind, rdt = self._router_args(router_logits, scores)
        self._ck(self.lib.b2m_route(self._h, layer, C.c_void_p(x2.data_ptr()),
                                    C.c_void_p(rin.data_ptr() if rin is not None else 0), kind, rdt, x2.shape[0],
                                    seq_len, C.c_void_p(_stream_ptr())))
        return x2.shape[0]

    def route_from_mask(self, layer: int, x: torch.Tensor, mask: torch.Tensor):
        x2 = self._check_x(x)
        m = mask.reshape(-1, self.E).to(self.device).ne(0).to(torch.uint8).contiguous()
        self._ck(self.lib.b2m_route_from_mask(self._h, layer, C.c_void_p(x2.data_ptr()), C.c_void_p(m.data_ptr()),
                                              x2.shape[0], C.c_void_p(_stream_ptr())))
        return x2.shape[0]

    def run_experts(self, layer: int, T: int, phases: int = 3):
        self._ck(self.lib.b2m_run_experts_ex(self._h, layer, T, phases, C.c_void_p(_stream_ptr())))

    def combine(self, layer: int, x: torch.Tensor, out: Optional[torch.Tensor] = None):
        x2 = self._check_x(x)
        if out is None:
            out = torch.empty_like(x2)
        self._ck(self.lib.b2m_combine(self._h, layer, C.c_void_p(x2.data_ptr()), x2.shape[0],
                                      C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr())))
        return out

    def expert_outputs(self, T: int):
        """(rows[T*k,H] model dtype grouped by ascending expert / ascending token, offsets list[E+1])."""
        rows = torch.empty(T * self.k, self.H, dtype=self.dtype, device=self.device)
        offs = (C.c_int * (self.E + 1))()
        self._ck(self.lib.b2m_expert_outputs(self._h, T, C.c_void_p(rows.data_ptr()), offs, C.c_void_p(_stream_ptr())))
        return rows, list(offs)

    def ws(self, name: str, T: int) -> torch.Tensor:
        """Zero-copy view of a workspace buffer, shaped for a call with T tokens."""
        p = C.c_void_p()
        self._ck(self.lib.b2m_ws_ptr(self._h, L.WS[name], C.byref(p)))
        k, E, H, I = self.k, self.E, self.H, self.I
        logits_dt = self.dtype if self.router in _MODEL_DTYPE_ROUTERS else torch.float32
        shape, dt = {
            "topk_idx": ((T, k), torch.int32), "topk_w": ((T, k), torch.float32), "row_of": ((T, k), torch.int32),
            "perm_token": ((T * k,), torch.int32), "counts": ((E,), torch.int32), "offsets": ((E + 1,), torch.int32),
            "xp": ((T * k, H), self.dtype), "hmid": ((T * k, I), self.dtype), "y": ((T * k, H), torch.float32),
            "scores": ((T, E), torch.float32), "logits": ((T, E), logits_dt),
            "shared_gate": ((T,), self.dtype), "y_shared": ((T, H), torch.float32),
        }[name]
        return _view(p.value, shape, dt, self.device)

    # ------------------------------------------------------------------ cache / prefetch
    @staticmethod
    def _pairs(pairs: Iterable[Tuple[int, int]]):
        flat = [int(v) for p in pairs for v in p]
        return (C.c_int32 * len(flat))(*flat), len(flat) // 2

    def replace_cache_candidates(self, pairs: Iterable[Tuple[int, int]]):
        arr, n = self._pairs(pairs)
        self._ck(self.lib.b2m_replace_cache_candidates(self._h, n, arr))

    def enqueue_prefetch(self, layer: int, expert: int):
        self._ck(self.lib.b2m_enqueue_prefetch(self._h, layer, expert))

    def prefetch_hint(self, pairs: Sequence[Tuple[int, int]], scores: Sequence[float]):
        arr, n = self._pairs(pairs)
        sc = (C.c_float * n)(*[float(s) for s in scores])
        self._ck(self.lib.b2m_prefetch_hint(self._h, n, arr, sc))

    def prefetch_pump(self):
        self._ck(self.lib.b2m_prefetch_pump(self._h))

    def prefetch_drain(self):
        self._ck(self.lib.b2m_prefetch_drain(self._h))

    def clear_expert_cache_counts(self):
        self._ck(self.lib.b2m_clear_expert_cache_counts(self._h))

    def is_resident(self, layer: int, expert: int) -> bool:
        r = self.lib.b2m_is_resident(self._h, layer, expert)
        if r < 0:
            self._ck(r)
        return bool(r)

    def stats(self) -> dict:
        s = L.Stats()
        self._ck(self.lib.b2m_stats_get(self._h, C.byref(s)))
        return s.as_dict()

    def last_lookahead(self) -> List[int]:
        arr = (C.c_int32 * self.E)()
        self._ck(self.lib.b2m_last_lookahead(self._h, arr))
        return list(arr)

    def last_counts(self) -> List[int]:
        arr = (C.c_int32 * self.E)()
        self._ck(self.lib.b2m_last_counts(self._h, arr))
        return list(arr)


class DecodeSession:
    """One decode step (all MoE layers of the model for a fixed batch) as a replayable CUDA graph with HOST I/O.

    The step's inputs live in pinned host memory (`x_host[L,T,H]`, written by the caller), the outputs come back in
    pinned host memory (`out_host[L,T,H]`); the graph contains the H2D copy, every layer's kernels and the D2H copy.
    Only valid when every expert is HBM resident (the on-demand path synchronises with the host and cannot be
    captured) -- which is exactly the regime where per-layer Python/launch overhead would otherwise matter."""

    def __init__(self, engine: MoEEngine, T: int, layers: Optional[Sequence[int]] = None):
        self.eng = engine
        self.layers = list(range(engine.L)) if layers is None else list(layers)
        n = len(self.layers)
        self.x_host = torch.zeros(n, T, engine.H, dtype=engine.dtype).pin_memory()
        self.out_host = torch.zeros(n, T, engine.H, dtype=engine.dtype).pin_memory()
        self._x = torch.zeros(n, T, engine.H, dtype=engine.dtype, device=engine.device)
        self._out = torch.zeros_like(self._x)
        self._graph = None

    def _run(self):
        self._x.copy_(self.x_host, non_blocking=True)
        for i, l in enumerate(self.layers):
            self.eng.forward(l, self._x[i], out=self._out[i])
        self.out_host.copy_(self._out, non_blocking=True)

    def capture(self):
        side = torch.cuda.Stream(device=self.eng.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._run()          # warm-up outside capture: kernel attributes, slot table upload
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._run()
        self._graph = g
        return self

    def step(self, sync: bool = True) -> torch.Tensor:
        """Replay the captured step on the current stream; returns the pinned output buffer."""
        if self._graph is None:
            self._run()
        else:
            self._graph.replay()
        if sync:
            torch.cuda.current_stream().synchronize()
        return self.out_host


class DeviceExpertTracer:
    """Device-side ExpertTracer + ExpertPredictor (moe_infinity/memory/expert_tracer.py:17-125, expert_predictor.py:7-35):
    the trace library and the per-sequence matrices live in HBM and one kernel per layer call does update_entry,
    find_most_similar and predict for every sequence of the batch -- no `.cpu()` in the layer (the reference pays two
    device syncs per sequence per layer).  Sequences are slots 0..max_seqs-1; a call's tokens are sequence-major
    (rows b*seq_len .. (b+1)*seq_len-1 belong to slot seq_slot0 + b; decode: seq_len = 1).
    Readers (`entry`, `prediction`, `hint`, `library`, `save_trace`) synchronise and are meant for tests / persistence."""

    def __init__(self, engine: MoEEngine, capacity: int, max_seqs: int, auto_prefetch: bool = False):
        self.eng, self.capacity, self.max_seqs = engine, capacity, max_seqs
        engine._ck(engine.lib.b2m_trace_init(engine._h, capacity, max_seqs, int(auto_prefetch)))

    def load_trace(self, trace):                       # expert_tracer.py:40-52
        import numpy as np
        if isinstance(trace, (str, bytes)) or hasattr(trace, "__fspath__"):
            trace = np.load(trace, allow_pickle=False)
        arr = np.ascontiguousarray(trace, dtype=np.float32)
        assert arr.shape[1:] == (self.eng.L, self.eng.E) and arr.shape[0] <= self.capacity
        self.eng._ck(self.eng.lib.b2m_trace_load(self.eng._h, arr.shape[0], C.c_void_p(arr.ctypes.data)))

    def create_entry(self, seq_slot: int):             # :54-59
        self.eng._ck(self.eng.lib.b2m_trace_reset_seq(self.eng._h, seq_slot, C.c_void_p(_stream_ptr())))
        return seq_slot

    def finish_entry(self, seq_slot: int):             # :61-76
        self.eng._ck(self.eng.lib.b2m_trace_finish_seq(self.eng._h, seq_slot, C.c_void_p(_stream_ptr())))

    def update_predict(self, layer: int, num_seqs: int, seq_len: int = 1, seq_slot0: int = 0):
        """update_entry + find_most_similar + predict for the routing call that just ran (asynchronous)."""
        self.eng._ck(self.eng.lib.b2m_trace_update_predict(self.eng._h, layer, seq_slot0, num_seqs, seq_len,
                                                           C.c_void_p(_stream_ptr())))

    def _read(self, what: int, index: int, n: int, dtype):
        import numpy as np
        out = np.zeros(n, dtype=dtype)
        self.eng._ck(self.eng.lib.b2m_trace_read(self.eng._h, what, index, C.c_void_p(out.ctypes.data)))
        return out

    def entry(self, seq_slot: int):
        import numpy as np
        return self._read(0, seq_slot, self.eng.L * self.eng.E, np.float32).reshape(self.eng.L, self.eng.E)

    def prediction(self, seq_slot: int):
        import numpy as np
        return self._read(1, seq_slot, self.eng.L * self.eng.E, np.float32).reshape(self.eng.L, self.eng.E)

    def hint(self):
        import numpy as np
        return self._read(2, 0, self.eng.L * self.eng.E, np.float32).reshape(self.eng.L, self.eng.E)

    def library(self, index: int):
        import numpy as np
        return self._read(3, index, self.eng.L * self.eng.E, np.float32).reshape(self.eng.L, self.eng.E)

    def access_counts(self):
        import numpy as np
        return self._read(4, 0, self.capacity, np.int32)

    def winner(self, seq_slot: int) -> int:
        import numpy as np
        return int(self._read(5, seq_slot, 1, np.int32)[0])

    def save_trace(self, path):
        """Persist the library (what `load_trace` reads back): np.save of [capacity][L][E] fp32."""
        import numpy as np
        np.save(path, np.stack([self.library(i) for i in range(self.capacity)]))
