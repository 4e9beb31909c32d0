"""Cases on which every expert GEMM has one exact answer -- shared by tests/test_gemm_exact_plans.py (CPU: launch plans,
coverage, reference) and tests/test_gpu_gemm_exact.py (GPU: the kernels against the reference with torch.equal).

The data: activations are dense integers in {1, 2, 3}; weights are sparse integers times a power of two (gate rows about 36
nonzeros of {1, 2}, up rows of {+-1, +-2}, down rows about 64 of {+-1}; the quantised formats reach the same values through
their codes and power-of-two scales).  Every output's sum |w * x| stays at or below 2^22 units (a unit = the product of the
two operands' smallest power-of-two steps), so every partial sum -- in any order, any split-K or stream-K grouping, any
order of the fp32 atomics and any operand alignment inside the tensor cores -- is an integer number of units that fp32
holds exactly.  Gate pre-activations stay in [32, 255] (so SiLU(g) = GELU(g) = ReLU(g) = g exactly: 1 + exp(-g) rounds to
1 and erf(g / sqrt 2) to 1) and up values within +-255, so g and u are exact in bf16 / f16 and a one-unit error in either
always shows in the 16-bit intermediate.  `reference` asserts all of this on the data it is given.

The reference sums in float64 on the caller's device, one expert and one matrix at a time (a full Mixtral matrix is 470 MB
in float64), and runs the elementwise chain with the torch dtype operations of oracle/moe_oracle.py:expert_ffn."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

SMS = 132                     # H100 SXM: the partition the stream-K plans below are stated for
BUDGET = 1 << 22              # units per output: two bits of headroom below fp32's 24-bit significand
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
NNZ = {"gate": 36, "up": 36, "down": 64}

MIXTRAL, DEEPSEEK, SWITCH, SWITCH_GATED, NLLB = "mixtral", "deepseek", "switch", "switch_gated", "nllb"
# include/b2m.h expert types
ETYPE = {SWITCH: 0, SWITCH_GATED: 1, NLLB: 2, MIXTRAL: 4, DEEPSEEK: 5}


@dataclass(frozen=True)
class Plan:
    """What the launch planner claims for a row: token-tile widths of K3 (gate/up) and K4 (down), split-K, stream-K,
    dual_m, early-A of each GEMM, and for stream-K rows the largest number of CTAs one K4 tile is spread over."""
    nt_up: int
    nt_dn: int
    splitk: bool
    stream_k: bool
    dual_m: bool
    early_up: bool
    early_dn: bool
    span: int = 0


@dataclass(frozen=True)
class Case:
    name: str
    etype: str
    H: int
    I: int
    E: int
    k: int
    dtype: str                 # model dtype: bf16 / f16 / f32
    fmt: str                   # A source: bf16 (model dtype), pk12 (12-bit packed copy), fp8, int4
    T: int
    counts: Tuple[int, ...]    # tokens per expert
    plan: Plan
    numerics: str = "reference"
    slots: int = 0             # 0 = every expert resident; else the HBM slot count (offload waves)
    shared: int = 0            # DeepSeek shared-expert intermediate size
    gemm_impl: int = 0         # 1 = the CUDA-core grouped GEMM

    @property
    def engine_key(self):
        """Rows with the same key share one engine (and its weights) on the GPU."""
        return (self.etype, self.H, self.I, self.E, self.k, self.dtype, self.fmt, self.numerics, self.slots, self.shared,
                self.gemm_impl)

    @property
    def routed_by_forward(self) -> bool:
        """Mixtral and DeepSeek rows route from designed router logits / scores through b2m_moe_forward; the Switch and
        NLLB rows route from a mask (b2m_route_from_mask) and run the experts with b2m_run_experts."""
        return self.etype in (MIXTRAL, DEEPSEEK)


def pick_nt(T: int) -> int:
    for nt in (16, 32, 64, 128):
        if T <= nt:
            return nt
    return 128


def design_counts(T: int, E: int, k: int, wish: Sequence[int] = ()) -> Tuple[int, ...]:
    """T * k rows over E experts, no expert above T: expert 0 takes every token (k > 1), expert 1 stays empty (E > 2), the
    counts in `wish` (tile width NT and NT + 1, say) go to experts 2, 3, ..., and the rest fills experts from the last
    one down."""
    c = [0] * E
    left = T * k
    if k > 1:
        c[0] = T
        left -= T
    nxt = 2 if E > 2 else 1
    for w in wish:
        if 0 < w <= min(T, left) and nxt < E:
            c[nxt] = w
            left -= w
            nxt += 1
    for e in range(E - 1, nxt - 1, -1):
        take = min(T - c[e], left)
        c[e] += take
        left -= take
    assert left == 0, (T, E, k, wish)
    return tuple(c)


def assignment(counts: Sequence[int], T: int, k: int) -> torch.Tensor:
    """int64 [T, k]: the experts of each token, k distinct ones, expert e chosen by counts[e] tokens.  The experts' rows
    are laid end to end and token t takes entries t, t + T, t + 2T, ...: an expert's run is at most T long, so no token
    meets one expert twice."""
    seq = [e for e, n in enumerate(counts) for _ in range(n)]
    assert len(seq) == T * k
    return torch.tensor(seq, dtype=torch.int64).reshape(k, T).t().contiguous()


def router_logits(counts: Sequence[int], T: int, k: int) -> torch.Tensor:
    """fp32 [T, E]: 10, 9, ... for a token's k experts and 0 elsewhere -- distinct margins, no ties."""
    idx = assignment(counts, T, k)
    lg = torch.zeros(T, len(counts))
    lg.scatter_(1, idx, (10.0 - torch.arange(k, dtype=torch.float32)).expand(T, k).contiguous())
    return lg


def route_mask(counts: Sequence[int], T: int, k: int) -> torch.Tensor:
    idx = assignment(counts, T, k)
    m = torch.zeros(T, len(counts), dtype=torch.bool)
    m.scatter_(1, idx, True)
    return m


# ------------------------------------------------------------------------------------------------ the case table
def _row(name, etype, H, I, E, k, dtype, fmt, T, plan, wish=None, counts=None, **kw) -> Case:
    if counts is None:
        nt = pick_nt(T)
        counts = design_counts(T, E, k, (nt, nt + 1) if wish is None else wish)
    return Case(name, etype, H, I, E, k, dtype, fmt, T, tuple(counts), plan, **kw)


MH, MI = 4096, 14336          # Mixtral-8x7B
CASES: List[Case] = []
for _fmt, _dt in (("bf16", "bf16"), ("pk12", "bf16"), ("fp8", "bf16"), ("int4", "bf16"), ("int4", "f16")):
    _tag = _fmt if _dt == "bf16" else f"{_fmt}_{_dt}"
    CASES += [
        _row(f"mixtral_{_tag}_T1", MIXTRAL, MH, MI, 8, 2, _dt, _fmt, 1, Plan(16, 16, True, True, False, True, True, 3)),
        _row(f"mixtral_{_tag}_T24", MIXTRAL, MH, MI, 8, 2, _dt, _fmt, 24, Plan(32, 32, True, True, False, True, True, 3)),
        _row(f"mixtral_{_tag}_T300", MIXTRAL, MH, MI, 8, 2, _dt, _fmt, 300, Plan(128, 128, True, True, True, False, False, 3)),
        _row(f"mixtral_{_tag}_T1100", MIXTRAL, MH, MI, 8, 2, _dt, _fmt, 1100, Plan(128, 256, True, True, False, False, False, 2)),
        # three m-tiles of the down matrix: one full dual_m pair and one whose second tile lies past the matrix
        _row(f"oddpair_{_tag}_T400", MIXTRAL, 384, 1024, 8, 2, _dt, _fmt, 400, Plan(128, 128, True, True, True, False, False, 8)),
    ]
CASES += [
    # ragged H and I (multiples of 8): M and K tails in both GEMMs, and a partial A0 with an out-of-range A1 under dual_m
    _row("ragged_bf16_T1", MIXTRAL, 328, 1416, 8, 2, "bf16", "bf16", 1, Plan(16, 16, True, True, False, True, True, 22)),
    _row("ragged_f16_T1", MIXTRAL, 328, 1416, 8, 2, "f16", "bf16", 1, Plan(16, 16, True, True, False, True, True, 22)),
    _row("ragged_bf16_T45", MIXTRAL, 328, 1416, 8, 2, "bf16", "bf16", 45, Plan(64, 64, True, True, False, True, True, 22)),
    _row("ragged_bf16_T400", MIXTRAL, 328, 1416, 8, 2, "bf16", "bf16", 400, Plan(128, 128, True, True, True, False, False, 8)),
    _row("ragged_f16_T400", MIXTRAL, 328, 1416, 8, 2, "f16", "bf16", 400, Plan(128, 128, True, True, True, False, False, 8)),
    # 16 (tile, k-block) units for 132 CTAs: most CTAs get none, the others fewer k-blocks than the ring has stages
    _row("small_bf16_T1", MIXTRAL, 128, 512, 8, 2, "bf16", "bf16", 1, Plan(16, 16, True, True, False, True, True, 8)),
    # one tile: a single expert row and one m-tile, its 224 k-blocks spread over every CTA
    _row("one_tile_T1", MIXTRAL, 128, MI, 8, 1, "bf16", "bf16", 1, Plan(16, 16, True, True, False, True, True, 132),
         counts=(1, 0, 0, 0, 0, 0, 0, 0)),
    # numerics fp32 (one rounding of act(g) * u), the fp32 CUDA-core path, the CUDA-core grouped GEMM, offload waves
    _row("mixtral_fp32num_T24", MIXTRAL, 1024, 2048, 8, 2, "bf16", "bf16", 24, Plan(32, 32, True, True, False, True, True, 9),
         numerics="fp32"),
    _row("mixtral_f32_T40", MIXTRAL, 256, 512, 8, 2, "f32", "bf16", 40, Plan(0, 0, False, False, False, False, False)),
    _row("mixtral_simt_T40", MIXTRAL, 256, 512, 8, 2, "bf16", "bf16", 40, Plan(0, 0, False, False, False, False, False),
         gemm_impl=1),
    _row("offload_T24", MIXTRAL, 512, 1024, 8, 2, "bf16", "bf16", 24, Plan(32, 32, True, True, False, False, True, 16),
         counts=(6, 6, 6, 6, 6, 6, 6, 6), slots=2),
    # DeepSeek-V2-Lite: 64 experts, top-6, the shared expert (2 x 1408) as a single-matrix tile table
    _row("deepseek_T1", DEEPSEEK, 2048, 1408, 64, 6, "bf16", "bf16", 1, Plan(16, 16, True, True, False, True, True, 3),
         shared=2816),
    _row("deepseek_T300", DEEPSEEK, 2048, 1408, 64, 6, "bf16", "bf16", 300, Plan(128, 128, False, False, True, False, False),
         shared=2816),
    # Switch (ReLU, one projection), Switch-gated (GELU), NLLB (biases, whole-K)
    _row("switch_T200", SWITCH, 768, 3072, 8, 1, "bf16", "bf16", 200, Plan(128, 128, True, True, True, False, False, 11),
         wish=(128, 129, 3, 1)),
    _row("switch_gated_T24", SWITCH_GATED, 768, 2048, 8, 2, "bf16", "bf16", 24, Plan(32, 32, True, True, False, False, True, 11)),
    _row("nllb_T40", NLLB, 512, 2048, 8, 2, "f16", "bf16", 40, Plan(64, 64, False, False, False, False, True)),
]
BY_NAME: Dict[str, Case] = {c.name: c for c in CASES}


# ------------------------------------------------------------------------------------------------ data
def matrix_shapes(etype: str, H: int, I: int):
    """(role, shape) of an expert's tensors in the order load_expert / expert_ffn take them."""
    return {MIXTRAL: [("gate", (I, H)), ("down", (H, I)), ("up", (I, H))],
            DEEPSEEK: [("gate", (I, H)), ("up", (I, H)), ("down", (H, I))],
            SWITCH_GATED: [("gate", (I, H)), ("up", (I, H)), ("down", (H, I))],
            SWITCH: [("gate", (I, H)), ("down", (H, I))],
            NLLB: [("gate", (I, H)), ("bias1", (I,)), ("down", (H, I)), ("bias2", (H,))]}[etype]


def _pow2(shape, lo, hi, g, dev):
    return torch.pow(2.0, torch.randint(lo, hi + 1, shape, generator=g, device=dev).double())


def _pattern(role, rows, cols, scaled, g, dev):
    """Sparse integer pattern: NNZ[role] nonzeros per row at random columns."""
    nnz = min(NNZ[role], cols)
    col = torch.randint(0, cols, (rows, nnz), generator=g, device=dev)
    mag = torch.ones(rows, nnz, device=dev, dtype=torch.float64)
    if role != "down" and not scaled:
        mag = mag + torch.randint(0, 2, (rows, nnz), generator=g, device=dev).double()     # {1, 2}
    if role != "gate":
        mag = mag * (torch.randint(0, 2, (rows, nnz), generator=g, device=dev).double() * 2 - 1)
    d = torch.zeros(rows, cols, device=dev, dtype=torch.float64)
    d.scatter_(1, col, mag)
    return d


@dataclass
class Expert:
    w: List[torch.Tensor]                             # dequantised tensors (what the GEMMs compute with), load order
    load: List[torch.Tensor] = field(default_factory=list)
    scales: Optional[List[torch.Tensor]] = None
    zeros: Optional[List[torch.Tensor]] = None


def make_expert(c: Case, seed: int, dev="cpu") -> Expert:
    """One expert's tensors in format c.fmt.  fp8: codes in {0, +-1} with a 2^j scale per 128x128 block; int4: s * (q - z)
    with s = 2^j per row and group of 128 inputs, z anywhere in 0..15 and q - z in {0, +-1}; bf16 / 12-bit packed copy:
    the plain integer recipe.  Gate and up scales 2^j take j in {0, 1}, down scales j in {-1, 0}."""
    g = torch.Generator(device=dev).manual_seed(seed)
    dt = DTYPES[c.dtype]
    scaled = c.fmt in ("fp8", "int4")
    ws, load, scales, zeros = [], [], [], []
    for role, shp in matrix_shapes(c.etype, c.H, c.I):
        if role.startswith("bias"):
            b = torch.randint(-2, 3, shp, generator=g, device=dev).to(dt)
            ws.append(b)
            load.append(b)
            continue
        rows, cols = shp
        d = _pattern(role, rows, cols, scaled, g, dev)
        lo, hi = (-1, 0) if role == "down" else (0, 1)
        if c.fmt == "fp8":
            s = _pow2((rows // 128, cols // 128), lo, hi, g, dev)
            w = d * s.repeat_interleave(128, 0).repeat_interleave(128, 1)
            load.append(d.float().to(torch.float8_e4m3fn))
            scales.append(s.float())
        elif c.fmt == "int4":
            grp = cols // 128
            s = _pow2((rows, grp), lo, hi, g, dev)
            z = torch.randint(0, 15 if role == "gate" else 16, (rows, grp), generator=g, device=dev)
            ze = z.repeat_interleave(128, 1).double()
            d = torch.where((ze + d > 15) | (ze + d < 0), -d, d)          # keep every code in 0..15
            w = d * s.repeat_interleave(128, 1)
            q = (ze + d).to(torch.uint8)
            load.append((q[:, 0::2] | (q[:, 1::2] << 4)).contiguous())
            scales.append(s.to(dt))
            zeros.append(z.to(torch.uint8))
        else:
            w = d
            load.append(d.to(dt))
        w = w.to(dt)
        ws.append(w)
    return Expert(ws, load, scales if scaled else None, zeros if c.fmt == "int4" else None)


def make_x(n: int, H: int, dtype: torch.dtype, seed: int, dev="cpu") -> torch.Tensor:
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(1, 4, (n, H), generator=g, device=dev).to(dtype)


def make_hmid(n: int, I: int, dtype: torch.dtype, seed: int, dev="cpu") -> torch.Tensor:
    """Dense small integers for the down projection alone."""
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(-3, 4, (n, I), generator=g, device=dev).to(dtype)


# ------------------------------------------------------------------------------------------------ reference
def _unit(t: torch.Tensor) -> float:
    """The largest power of two (<= 1) every value of t is an integer multiple of."""
    u = 1.0
    t = t.double()
    while not bool((torch.remainder(t, u) == 0).all()):
        u /= 2
        assert u >= 2.0 ** -30, "operand values are not small binary fractions"
    return u


def exact_linear(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """x @ w.T in float64, after checking that every partial sum is exact in fp32: sum |w x| <= 2^22 units."""
    xd, wd = x.double(), w.double()
    ux, uw = _unit(xd), _unit(wd)
    worst = (xd.abs() @ wd.abs().t()).max().item() if x.shape[0] else 0.0
    assert worst <= BUDGET * ux * uw, f"budget: {worst / (ux * uw):.0f} units > 2^22"
    return xd @ wd.t()


def _exact_in(v: torch.Tensor, dt: torch.dtype, what: str) -> torch.Tensor:
    r = v.to(dt)
    assert torch.equal(r.double(), v.double()), f"{what} is not exact in {dt}"
    return r


def reference(c: Case, x: torch.Tensor, w: Sequence[torch.Tensor], hmid: Optional[torch.Tensor] = None):
    """(hmid [n, I] model dtype, y [n, H] fp32) of one expert on rows x.  With `hmid` given, only the down projection
    of those rows.  y is what the down GEMM leaves in the workspace: the exact sum (NLLB: rounded, + fc2_bias, rounded)."""
    dt = DTYPES[c.dtype]
    ws = dict(zip([r for r, _ in matrix_shapes(c.etype, c.H, c.I)], w))
    if hmid is None:
        g = exact_linear(x, ws["gate"])
        assert g.numel() == 0 or bool((g >= 32).all()), "a gate pre-activation below 32: act(g) would not be g"
        limit = 2047 if dt == torch.float16 else 255
        assert g.numel() == 0 or g.abs().max().item() <= limit
        gd = _exact_in(g, dt, "g")
        if c.etype == NLLB:
            # relu(matmul(x, fc1^T) + fc1_bias): g + b >= 30 and exact in the model dtype
            _exact_in(gd.double() + ws["bias1"].double(), dt, "g + b1")
            hmid = torch.relu(gd + ws["bias1"])
        elif c.etype == SWITCH:
            hmid = torch.relu(gd)
        else:
            u = exact_linear(x, ws["up"])
            assert u.numel() == 0 or u.abs().max().item() <= limit
            ud = _exact_in(u, dt, "u")
            act = F.gelu(gd) if c.etype == SWITCH_GATED else F.silu(gd)
            assert torch.equal(act, gd), "act(g) != g"
            if c.numerics == "fp32" or dt == torch.float32:
                hmid = (gd.double() * ud.double()).to(dt)       # one rounding of act(g) * u
            else:
                hmid = act * ud
    y = exact_linear(hmid, ws["down"])
    if c.etype == NLLB:
        y = (y.to(dt) + ws["bias2"]).double()
    y32 = y.float()
    assert torch.equal(y32.double(), y), "y is not exact in fp32"
    return hmid, y32


def stream_k_spans(units_per_tile: int, tiles: int, sms: int = SMS) -> List[int]:
    """CTAs each tile's units are spread over when CTA b takes units [units * b / sms, units * (b + 1) / sms) (gemm_body)."""
    units = units_per_tile * tiles
    bounds = [units * b // sms for b in range(sms + 1)]
    out = []
    for t in range(tiles):
        lo, hi = t * units_per_tile, (t + 1) * units_per_tile
        out.append(sum(1 for b in range(sms) if bounds[b] < bounds[b + 1] and bounds[b] < hi and bounds[b + 1] > lo))
    return out


def expert_rows(counts: Sequence[int], T: int, k: int) -> List[torch.Tensor]:
    """Tokens of each expert in ascending token order (the row order of the grouped GEMMs)."""
    idx = assignment(counts, T, k)
    return [torch.nonzero((idx == e).any(dim=1)).flatten() for e in range(len(counts))]
