"""Expert parallelism with every rank in one process on one GPU: N MoEEngine contexts, one per simulated rank, each holding
only its own experts, and the all-to-all of ep.py replaced by tensor copies on the current stream.  The buffer entry points
(b2m_ep_pack / regroup / ungroup / unpack) take plain device pointers and a stream, so the four exchange kernels of
csrc/ep.cu run here exactly as they run between GPUs -- no NCCL, no IPC, no second device.

* `LoopbackEP` drives one step (route -> pack -> exchange -> regroup -> run_experts -> ungroup -> exchange back -> unpack
  -> combine, per layer) in either counts layout, with a caller-chosen capacity and one T_local per rank.  `fill_sentinels`
  fills every exchange buffer with a NaN bit pattern (the GPU test does so before each layer), so a row a kernel reads
  but nobody wrote shows up downstream.
* `expected_exchange` states the exchange contract of ep.cu's header in plain Python: which rows each source sends to each
  owner, in which slots, and where each owner puts them.
* `CASES` is the table of rows tests/test_gpu_ep_loopback.py runs and tests/test_ep_loopback_cases.py checks on the CPU;
  each row names what it exists for."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

import gemm_exact_cases as X

SENTINEL = 0x7FA5                 # a NaN in both bf16 and f16 (all-ones exponent, nonzero mantissa)
COUNT_SENTINEL = -0x5A5A5A5B      # what an unwritten separate-layout counts entry holds
INLINE, SEPARATE = "inline", "separate"
# router kinds of the rows (include/b2m.h B2M_ROUTER_*)
MIXTRAL, GREEDY, GROUP, SWITCH, V3 = "mixtral", "greedy", "group", "switch", "deepseek_v3"
ROUTER_ID = {MIXTRAL: 0, GREEDY: 1, GROUP: 2, SWITCH: 3, V3: 4}
ETYPE_OF = {MIXTRAL: X.MIXTRAL, GREEDY: X.DEEPSEEK, GROUP: X.DEEPSEEK, SWITCH: X.SWITCH, V3: X.DEEPSEEK}


# ------------------------------------------------------------------------------------------------ designed routing
def spread(T: int, k: int, experts: Sequence[int], E: int) -> Tuple[int, ...]:
    """Per-expert counts over E experts: T * k rows as evenly as possible over `experts` (at least k of them), none above T."""
    assert len(experts) >= k and len(set(experts)) == len(experts)
    c = [0] * E
    base, extra = divmod(T * k, len(experts))
    for i, e in enumerate(experts):
        c[e] = base + (1 if i < extra else 0)
    assert max(c) <= T and sum(c) == T * k
    return tuple(c)


def rotated(counts: Sequence[int], by: int) -> Tuple[int, ...]:
    E = len(counts)
    return tuple(counts[(e - by) % E] for e in range(E))


Design = Callable[[int, int, int, int, int], Optional[Tuple[int, ...]]]   # (layer, rank, T, E, k) -> counts or None


def _d_full_t1(l, r, T, E, k):
    return spread(T, k, [[0, 1], [2, 5]][r] if l == 0 else [[7, 3], [4, 6]][r], E)


def _d_full_f16(l, r, T, E, k):
    if l == 0:   # rank 1 sends all T * k rows to owner 0: a full peer segment
        return spread(T, k, list(range(E)) if r == 0 else [0, 1, 2, 3], E)
    return spread(T, k, [4, 5, 6, 7], E) if r == 0 else X.design_counts(T, E, k)


def _d_n8(l, r, T, E, k):
    if l == 0:
        return spread(T, k, [(r + j) % E for j in range(4)], E)
    return rotated(X.design_counts(T, E, k), r)


def _d_prefill(l, r, T, E, k):
    if l == 0:   # nobody routes to experts 6 and 7: their owner (rank 3) receives nothing
        return spread(T, k, [0, 1, 2, 3, 4, 5], E)
    return rotated(X.design_counts(T, E, k, (128, 129)), 2 * r)


def _d_deepseek(l, r, T, E, k):
    return spread(T, k, sorted({(8 * r + 3 * j) % E for j in range(12)}), E)


def _d_group(l, r, T, E, k):
    # every token's experts inside groups r, r+1, r+2 (8 experts per group): the top-3 groups keep all of them
    return spread(T, k, sorted({(8 * ((r + g) % 8) + j) for g in range(3) for j in (0, 3, 5, 6)}), E)


def _d_e256(l, r, T, E, k):
    # both sources route to the first and last expert of each owner, and each to 12 experts of its own
    ex = [0, 127, 128, 255] + [(97 * r + 13 * j) % E for j in range(1, 13)]
    return spread(T, k, ex, E)


def _d_e64(l, r, T, E, k):
    return spread(T, k, sorted({(4 * r + 5 * j) % E for j in range(8)}), E)


def _d_uneven(l, r, T, E, k):
    if T == 0:
        return tuple([0] * E)
    if l == 0:
        return spread(T, k, [(2 * r + j) % E for j in range(3 if T > 1 else 2)], E)
    return rotated(X.design_counts(T, E, k), 3 * r)


# ------------------------------------------------------------------------------------------------ the case table
@dataclass(frozen=True)
class EpCase:
    name: str
    router: str
    H: int
    I: int
    E: int
    k: int
    dtype: str
    N: int
    steps: Tuple[Tuple[int, ...], ...]      # T_local of every rank, one tuple per step
    layouts: Tuple[str, ...]                # counts layout of each step (the last one repeats)
    why: str
    layers: int = 1
    cap: int = 0                            # 0: the largest T_local * k of the row
    shared: int = 0
    n_group: int = 1
    topk_group: int = 1
    expert_capacity: int = 0
    design: Optional[Design] = None         # None: routing from random logits, taken from the engine

    @property
    def El(self) -> int:
        return self.E // self.N

    @property
    def etype(self) -> str:
        return ETYPE_OF[self.router]

    @property
    def capacity(self) -> int:
        return self.cap or max(max(s) for s in self.steps) * self.k

    @property
    def max_tokens(self) -> int:
        """What the contexts are created with: ep_check needs N * cap rows (max_tokens * k) in the workspace."""
        return max(16, -(-self.N * self.capacity // self.k))

    def layout(self, step: int) -> str:
        return self.layouts[min(step, len(self.layouts) - 1)]

    def expert_case(self, T: int = 1) -> X.Case:
        """The gemm_exact_cases row whose data and reference these experts use."""
        return X.Case(self.name, self.etype, self.H, self.I, self.E, self.k, self.dtype, "bf16", T, (T * self.k,),
                      X.Plan(0, 0, False, False, False, False, False))

    def shared_case(self) -> X.Case:
        return X.Case("shared", X.DEEPSEEK, self.H, self.shared, 1, 1, self.dtype, "bf16", 1, (1,),
                      X.Plan(0, 0, False, False, False, False, False))


MH, MI = X.MH, X.MI
CASES: List[EpCase] = [
    EpCase("mixtral_full_n2_t1", MIXTRAL, MH, MI, 8, 2, "bf16", 2, ((1, 1), (1, 1)), (INLINE,),
           "T_total = 2: the owner's down GEMM runs split-K, so regroup's clear of y matters", layers=2, design=_d_full_t1),
    EpCase("mixtral_full_n2_f16", MIXTRAL, MH, MI, 8, 2, "f16", 2, ((12, 12),), (INLINE,),
           "the f16 ungroup / unpack instantiations; a full peer segment", layers=2, design=_d_full_f16),
    EpCase("mixtral_n8_el1", MIXTRAL, 1024, 2048, 8, 2, "bf16", 8, ((24,) * 8,), (SEPARATE,),
           "one expert per rank; the separate counts layout", layers=2, design=_d_n8),
    EpCase("mixtral_n4_prefill", MIXTRAL, 1024, 2048, 8, 2, "bf16", 4, ((300,) * 4,), (INLINE,),
           "multi-CTA routing on each rank; T_total = 1200, 2400 regroup slots over the grid-stride loop; a rank that "
           "receives nothing and experts nobody routes to", layers=2, design=_d_prefill),
    EpCase("deepseek_lite_n8_shared", GREEDY, 2048, 1408, 64, 6, "bf16", 8, ((8,) * 8,), (INLINE,),
           "the shared expert, which runs locally in each rank's combine", shared=2816, design=_d_deepseek),
    EpCase("deepseek_group_n4", GROUP, 512, 1024, 64, 6, "bf16", 4, ((40,) * 4,), (SEPARATE,),
           "the group router under EP", n_group=8, topk_group=3, design=_d_group),
    EpCase("e256_n2_el128", GREEDY, 512, 512, 256, 8, "bf16", 2, ((16, 16),), (INLINE,),
           "128 experts per rank (EP_MAX_EL); inline counts at exactly 4E = 2H", design=_d_e256),
    EpCase("e64_n16", GREEDY, 256, 128, 64, 6, "bf16", 16, ((4,) * 16, (4,) * 16), (INLINE, SEPARATE),
           "16 ranks (EP_MAX_RANKS); both layouts on the same contexts; I = 128 (two k-blocks): a whole-K owner plan, "
           "where regroup clears nothing", design=_d_e64),
    EpCase("v3_n8", V3, 512, 512, 256, 8, "bf16", 8, ((8,) * 8,), (INLINE,),
           "the DeepSeek-V3 router with its correction bias under EP", n_group=8, topk_group=4),
    EpCase("switch_n4_drop", SWITCH, 768, 3072, 8, 1, "bf16", 4, ((32,) * 4,), (INLINE,),
           "Switch capacity drops (topk_idx = -1): fewer rows than T_local * k; the pass-through combine",
           expert_capacity=3),
    EpCase("uneven_n4", MIXTRAL, 512, 1024, 8, 2, "bf16", 4, ((1, 37, 0, 16), (16, 0, 37, 1)), (INLINE,),
           "uneven and zero T_local; cap with slack; two steps on the same contexts", layers=2, cap=40 * 2,
           design=_d_uneven),
]
BY_NAME: Dict[str, EpCase] = {c.name: c for c in CASES}


# ------------------------------------------------------------------------------------------------ the exchange contract
@dataclass
class Exchange:
    send: List[List[List[int]]]          # send[s][r]: source s's tokens bound for owner r, in slot order
    counts: List[List[int]]              # counts[s][e]: rows source s routed to expert e
    offsets: List[List[int]]             # offsets[r]: owner r's offsets over global expert ids (E + 1)
    token: List[List[Tuple[int, int]]]   # token[r][i]: (source, token) of owner r's workspace row i
    slot: List[List[Tuple[int, int]]]    # slot[r][i]: (source, slot) that row i came from
    expert: List[List[int]]              # expert[r][i]: global expert of row i


def expected_exchange(topk_idx: Sequence[torch.Tensor], N: int, E: int) -> Exchange:
    """The exchange of ep.cu's header for each rank's routing topk_idx[s] ([T_s, k], -1 = dropped).  A source's rows are its
    routed (token, expert) pairs sorted by expert, then token; the ones of owner r's experts are contiguous and fill slots
    0, 1, ... of the segment for r.  Owner r takes them expert-major, then by source rank, then in source token order."""
    El = E // N
    rows = []                                                   # rows[s]: (expert, token) in source order
    for idx in topk_idx:
        pairs = [(int(e), t) for t, row in enumerate(idx.tolist()) for e in row if e >= 0]
        rows.append(sorted(pairs))
    counts = [[sum(1 for e, _ in rs if e == x) for x in range(E)] for rs in rows]
    send = [[[t for e, t in rs if e // El == r] for r in range(N)] for rs in rows]
    offsets, token, slot, expert = [], [], [], []
    for r in range(N):
        tok, sl, ex = [], [], []
        for e in range(r * El, (r + 1) * El):
            for s in range(N):
                seg = [(e2, t) for e2, t in rows[s] if e2 // El == r]
                for c, (e2, t) in enumerate(seg):
                    if e2 == e:
                        tok.append((s, t))
                        sl.append((s, c))
                        ex.append(e)
        off = [0] * (E + 1)
        for e in range(E + 1):
            off[e] = sum(1 for x in ex if x < e)
        offsets.append(off)
        token.append(tok)
        slot.append(sl)
        expert.append(ex)
    return Exchange(send, counts, offsets, token, slot, expert)


# ------------------------------------------------------------------------------------------------ the driver
def router_input(c: EpCase, layer: int, rank: int, T: int, seed: int):
    """(router_logits, scores) for one rank's tokens: designed (the gemm_exact_cases recipe) or random fp32 logits.  Always
    at least one row allocated, so that a rank without tokens still hands the routing call a valid pointer."""
    g = torch.Generator().manual_seed(seed)
    counts = c.design(layer, rank, T, c.E, c.k) if c.design else None
    if counts is not None and T > 0:
        lg = X.router_logits(counts, T, c.k)
    else:
        lg = torch.randn(max(T, 1), c.E, generator=g)
    lg = torch.cat([lg, torch.zeros(max(0, 1 - lg.shape[0]), c.E)])
    if c.router in (GREEDY, GROUP) and counts is not None:
        return None, torch.softmax(lg, dim=-1)
    return lg, None


class LoopbackEP:
    """N engines, rank r holding experts [r * El, (r + 1) * El) of every layer; one step runs every rank's calls in turn on
    the current stream and moves rows between their exchange buffers with tensor copies."""

    def __init__(self, c: EpCase, make_engine: Callable[[Optional[int]], object]):
        from moe_infinity_b200.ep import _EngineOps
        self.c = c
        self.engines = [make_engine(r) for r in range(c.N)]
        self.ops = [_EngineOps(e) for e in self.engines]
        self.bufs: Dict[Tuple[str, int], Dict[str, torch.Tensor]] = {}

    def close(self):
        for e in self.engines:
            e.close()
        self.engines, self.ops, self.bufs = [], [], {}

    def buffers(self, layout: str, cap: int) -> Dict[str, torch.Tensor]:
        """send / recv / ret / back [N ranks][N peers][rows][H] (rows = cap + 1 inline, cap separate) and, separate,
        send_counts [N][E] and recv_counts [N][N][E]."""
        key = (layout, cap)
        if key not in self.bufs:
            c, dev = self.c, self.engines[0].device
            dt = X.DTYPES[c.dtype]
            rows = cap + 1 if layout == INLINE else cap
            b = {n: torch.empty(c.N, c.N, rows, c.H, dtype=dt, device=dev) for n in ("send", "recv", "ret", "back")}
            if layout == SEPARATE:
                b["send_counts"] = torch.empty(c.N, c.E, dtype=torch.int32, device=dev)
                b["recv_counts"] = torch.empty(c.N, c.N, c.E, dtype=torch.int32, device=dev)
            self.bufs[key] = b
        return self.bufs[key]

    def fill_sentinels(self, b: Dict[str, torch.Tensor]):
        for n in ("send", "recv", "ret", "back"):
            b[n].view(torch.int16).fill_(SENTINEL)
        for n in ("send_counts", "recv_counts"):
            if n in b:
                b[n].fill_(COUNT_SENTINEL)

    def layer(self, layer: int, xs: Sequence[torch.Tensor], rins: Sequence[Tuple], outs: Sequence[torch.Tensor],
              layout: str, cap: int, probe: Optional[Callable[[str], None]] = None):
        """One expert-parallel layer over every rank.  rins[r] = (router_logits, scores) of rank r (rows past T_local are
        not read); probe(phase) runs after each phase of all ranks."""
        c, N = self.c, self.c.N
        b = self.buffers(layout, cap)
        Ts = [x.shape[0] for x in xs]
        T_total = sum(Ts)
        sep = layout == SEPARATE
        for r, e in enumerate(self.engines):
            lg, sc = rins[r]
            e.route(layer, xs[r], router_logits=None if lg is None else lg[:Ts[r]],
                    scores=None if sc is None else sc[:Ts[r]], seq_len=Ts[r] if c.router == SWITCH else 0)
        for r, o in enumerate(self.ops):
            o.pack(N, r, cap, Ts[r], b["send"][r], b["send_counts"][r] if sep else None)
        probe and probe("pack")
        b["recv"].copy_(b["send"].transpose(0, 1))                           # recv_r[s] = send_s[r]
        if sep:
            b["recv_counts"].copy_(b["send_counts"].unsqueeze(0).expand(N, N, c.E))
        for r, o in enumerate(self.ops):
            o.regroup(N, r, cap, T_total, b["recv"][r], b["recv_counts"][r] if sep else None)
        probe and probe("regroup")
        for r, o in enumerate(self.ops):
            o.run_experts(layer, T_total)
        for r, o in enumerate(self.ops):
            o.ungroup(N, r, cap, b["ret"][r])
        probe and probe("ungroup")
        b["back"].copy_(b["ret"].transpose(0, 1))                            # back_s[r] = ret_r[s]
        for r, o in enumerate(self.ops):
            o.unpack(N, r, cap, Ts[r], b["back"][r])
        probe and probe("unpack")
        for r, e in enumerate(self.engines):
            e.combine(layer, xs[r], out=outs[r])
        probe and probe("combine")
