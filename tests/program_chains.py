"""The chains of tests/test_gpu_program_chains.py: decode programs whose segments hold several ops of the persistent kernel
(csrc/decode_program.cuh), and a host restatement of what each chain reaches there. Importable without a GPU.

A chain is a list of op calls over named buffers. The GPU test records it twice: as it is, and with a separator (one tiny
plain launch on private scratch) after every persistent-capable call, so that each persistent op runs in a segment of its
own. Each op's plan depends only on its own shape, the grid and the workspace (sk_plan below), the split reduction runs in
fixed order and the glue ops are per row or per element, so both programs must give the same bits.

The restatements cite the code they mirror; tests/test_program_chains.py pins them on inputs that take every branch:
- sk_plan: c_api.cu:238 (the persistent kernel's split-K plan);
- SegCfg: decode_program.cuh:133 and wo_gemm.cuh:56-62 (ring depths, shared memory, CTAs per SM);
- sk_range and the ring counters: decode_program.cuh:161 (a CTA's k-block run), :170-215 (the producers' counters cw, cx)
  and :222-387 (the consumer's counter cb);
- rec_segment_op: c_api.cu:325 (which calls share a segment)."""
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

BK = 128                      # kGemmBK: k elements per block
TILE_N = 128                  # kGemmTileN: output features per tile
SEG_THREADS, DQ_THREADS = 320, 256
SEG_NORM_MAX_HIDDEN = 8192    # kSegNormMaxHidden: wider norms are their own launch
SEM_BYTES = 16384 + 2048 * 4  # kGemmSemBytes: the counters at the head of the GEMM workspace, partials after them
W_BYTES = {"int4": 8192 + 256 + 256, "int8": 16384}
SMS = 132                     # an H100 SXM
SMEM_PER_SM = 227 * 1024


# ---------------------------------------------------------------------------------------------- restated host / kernel arithmetic
def bpad_of(B: int) -> int:
    """gemm_bpad (c_api.cu:189)."""
    return 16 if B <= 16 else (32 if B <= 32 else (64 if B <= 64 else 128))


def sk_plan(n_tiles: int, k_blocks: int, grid: int, bpad: int, ws_partial_bytes: float = float("inf")) -> int:
    """Run length (k-blocks per CTA) of the persistent kernel's split-K plan, c_api.cu:238."""
    total = n_tiles * k_blocks
    slot = bpad * TILE_N * 4
    want = -(-total // grid)
    if want >= k_blocks:
        return -(-want // k_blocks) * k_blocks          # whole tiles, possibly several per CTA
    for d in range(want, k_blocks + 1):
        S = k_blocks // d
        if k_blocks % d == 0 and (S & (S - 1)) == 0 and S <= 16 and n_tiles * S * slot <= ws_partial_bytes:
            return d
    return k_blocks


def split_of(k_blocks: int, per: int) -> int:
    """S, the contributors of a tile: 1 for whole tiles."""
    return k_blocks // per if per < k_blocks else 1


def seg_cfg(fmt: str, bpad: int) -> dict:
    """SegCfg<FMT, BPAD>: activation stages XS, weight stages WS, dynamic shared memory, CTAs per SM."""
    xs = 4 if bpad <= 32 else 3
    x_bytes = bpad * 256
    ws = min(12, (106 * 1024 - 2048 - xs * x_bytes) // W_BYTES[fmt])
    smem = xs * x_bytes + ws * W_BYTES[fmt] + 2048
    return dict(XS=xs, WS=ws, SMEM=smem, per_sm=2 if 2 * (smem + 1024) <= SMEM_PER_SM else 1)


def segment_grid(fmt: str, bpad: int, sms: int = SMS) -> int:
    """segment_inst.cuh:46: every CTA co-resident, at most 2 per SM."""
    return seg_cfg(fmt, bpad)["per_sm"] * sms


def sk_run(n_tiles: int, k_blocks: int, per: int, cta: int) -> Tuple[int, int]:
    """sk_range: the CTA's global k-block range [g0, g1) (decode_program.cuh:161)."""
    total = n_tiles * k_blocks
    return min(cta * per, total), min(cta * per + per, total)


# ---------------------------------------------------------------------------------------------- chains
@dataclass(frozen=True)
class Op:
    """One op call. kind: gemm (x -> y, weight fmt / K / N, bias, fused SiLU*mul), norm (x [+ res in place] -> y, hidden),
    rope (qkv x -> q y, appends into the case's pool through its page list `pl` at `seq`), embed (ids x -> y), table
    (block ids x -> page list y), attn (q x -> y over the case's pool; always its own launch)."""
    kind: str
    x: str
    y: str
    fmt: str = ""
    K: int = 0
    N: int = 0
    bias: bool = False
    silu: bool = False
    res: Optional[str] = None
    hidden: int = 0

    def reads(self) -> Tuple[str, ...]:
        extra = {"norm": (self.res,) if self.res else (), "rope": ("pool", "pl", "seq"), "attn": ("pool", "pl", "seq")}
        return (self.x,) + extra.get(self.kind, ())

    def writes(self) -> Tuple[str, ...]:
        return (self.y,) + ((self.res,) if self.kind == "norm" and self.res else ()) + (("pool",) if self.kind == "rope" else ())


def gemm(x, y, fmt, K, N, bias=False, silu=False):
    return Op("gemm", x, y, fmt=fmt, K=K, N=N, bias=bias, silu=silu)


def norm(x, y, hidden, res=None):
    return Op("norm", x, y, hidden=hidden, res=res)


def rope(qkv, q):
    return Op("rope", qkv, q)


def embed(ids, y, hidden):
    return Op("embed", ids, y, hidden=hidden)


def table(bid, pl):
    return Op("table", bid, pl)


def attn(q, y):
    return Op("attn", q, y)


@dataclass(frozen=True)
class Chain:
    name: str
    dtype: str                     # "f16" | "bf16"
    B: int
    ops: Tuple[Op, ...]
    claims: Tuple[str, ...] = ()   # what coverage() must report for this chain (see CLAIMS)
    Hq: int = 8
    Hkv: int = 2
    D: int = 128
    T: int = 16
    M: int = 4                     # pages per sequence
    vocab: int = 1000              # rows of the embedding table


def persistent(op: Op, B: int) -> bool:
    """Whether the call is an op of the persistent kernel inside a program (c_api.cu: wo_gemm_impl :726, b200_add_rmsnorm :823,
    rope_append_impl :923, b200_embedding :1002, b200_convert_block_table :391)."""
    if op.kind == "gemm":
        return op.fmt in ("int4", "int8") and bpad_of(B) <= 64
    if op.kind == "norm":
        return op.hidden <= SEG_NORM_MAX_HIDDEN
    return op.kind in ("rope", "embed", "table")


def segment_key(op: Op, chain: Chain) -> Tuple[int, int, int]:
    """(bf16, bpad, qfmt) of rec_segment_op, -1 where the op does not care."""
    bf16 = int(chain.dtype == "bf16")
    if op.kind == "gemm":
        return bf16, bpad_of(chain.B), {"int8": 1, "int4": 2}[op.fmt]     # B200_FMT_INT8 / B200_FMT_INT4
    if op.kind in ("norm", "rope"):
        return bf16, -1, -1
    return -1, -1, -1


def segments(chain: Chain) -> List[dict]:
    """The launches a recording of the chain makes (rec_segment_op, c_api.cu:325): {"ops": [op indices]} for a segment,
    {"plain": op index} for a call that is its own launch."""
    items: List[dict] = []
    for i, op in enumerate(chain.ops):
        if not persistent(op, chain.B):
            items.append({"plain": i})
            continue
        k = segment_key(op, chain)
        last = items[-1] if items else None
        if last and "ops" in last and all(a < 0 or b < 0 or a == b for a, b in zip(last["key"], k)):
            last["key"] = tuple(a if a >= 0 else b for a, b in zip(last["key"], k))
            last["ops"].append(i)
        else:
            items.append({"ops": [i], "key": k})
    for it in items:
        if "ops" in it:
            bf16, bpad, qfmt = it["key"]
            it["bpad"] = bpad if bpad > 0 else 32             # b200_program_launch's defaults for a glue-only segment
            it["fmt"] = {1: "int8", 2: "int4"}.get(qfmt, "int4")
    return items


def n_tiles(op: Op) -> int:
    return -(-op.N // TILE_N)


def glue_busy(op: Op, chain: Chain, grid: int) -> int:
    """CTAs with work in a glue op: norm and embedding take rows, rope and the block table flatten over 256 dq threads."""
    if op.kind in ("norm", "embed"):
        return min(chain.B, grid)
    if op.kind == "rope":
        units = chain.B * (chain.Hq + 2 * chain.Hkv) * (chain.D // 2)
    else:
        units = chain.B * chain.M
    return min(grid, -(-units // DQ_THREADS))


def coverage(chain: Chain, grid: Optional[int] = None) -> dict:
    """What the chain reaches in the persistent kernel, at `grid` CTAs per segment (default: segment_grid of the segment).

    Per op (index into chain.ops): "segment", "pos" (the op's index in its segment), "idle" CTAs; a GEMM adds "per", "S",
    "tiles_per_cta", and "rings": the sorted set of ring states a CTA with work starts the op in, each
    (weight slot, weight phase, activation slot, activation phase); the consumer's counter cb equals the producers' cw and
    cx at every op start (all three advance by g1 - g0 per GEMM), so it reads the same weight and activation slots.
    Chain-wide: "glue_after_idle" (glue op, idle CTAs of the GEMM before it), "split_pairs" (two split GEMMs one after the
    other in a segment: first, second, S of each, tiles both use), "war" (an op writing a buffer the op before it in the same
    segment read), "segments" (ops per launch, None for a plain launch)."""
    out: Dict = dict(ops={}, glue_after_idle=[], split_pairs=[], war=[], segments=[])
    for si, it in enumerate(segments(chain)):
        if "plain" in it:
            out["segments"].append(None)
            continue
        fmt, bpad = it["fmt"], it["bpad"]
        G = grid or segment_grid(fmt, bpad)
        cfg = seg_cfg(fmt, bpad)
        counter = [0] * G                                     # cw == cx == cb of every CTA
        prev_gemm = None
        out["segments"].append(len(it["ops"]))
        for pos, i in enumerate(it["ops"]):
            op = chain.ops[i]
            rec = dict(segment=si, pos=pos)
            if op.kind == "gemm":
                kb, nt = op.K // BK, n_tiles(op)
                per = sk_plan(nt, kb, G, bpad)
                rings = set()
                busy = 0
                for c in range(G):
                    g0, g1 = sk_run(nt, kb, per, c)
                    if g1 > g0:
                        busy += 1
                        n = counter[c]
                        rings.add((n % cfg["WS"], (n // cfg["WS"]) & 1, n % cfg["XS"], (n // cfg["XS"]) & 1))
                    counter[c] += g1 - g0
                S = split_of(kb, per)
                rec.update(per=per, S=S, tiles_per_cta=per // kb if per >= kb else 0, idle=G - busy, rings=sorted(rings))
                if S > 1 and prev_gemm is not None and out["ops"][prev_gemm]["S"] > 1:
                    out["split_pairs"].append((prev_gemm, i, out["ops"][prev_gemm]["S"], S,
                                               min(nt, n_tiles(chain.ops[prev_gemm]))))
                prev_gemm = i
            else:
                rec["idle"] = G - glue_busy(op, chain, G)
                if pos > 0 and chain.ops[it["ops"][pos - 1]].kind == "gemm":
                    out["glue_after_idle"].append((i, out["ops"][it["ops"][pos - 1]]["idle"]))
            if pos > 0:
                before = chain.ops[it["ops"][pos - 1]]
                hit = set(op.writes()) & set(before.reads())
                if hit:
                    out["war"].append((it["ops"][pos - 1], i, sorted(hit)))
            out["ops"][i] = rec
    return out


def mid_ring_phase1(cov: dict) -> Dict[str, bool]:
    """Whether some GEMM starts, in some CTA with work, at a nonzero slot with phase 1 of the weight ring, of the activation
    ring, and (the same counter) of the consumer's view of both."""
    w = x = False
    for rec in cov["ops"].values():
        for ws, wp, xs, xp in rec.get("rings", ()):
            w |= ws != 0 and wp == 1
            x |= xs != 0 and xp == 1
    return dict(weight=w, activation=x, consumer=w and x)


CLAIMS = {   # claim: predicate over coverage()
    "idle>250 then glue": lambda c: any(n > 250 for _, n in c["glue_after_idle"]),
    "several tiles per CTA": lambda c: any(r.get("tiles_per_cta", 0) > 1 for r in c["ops"].values()),
    "S16 then S2": lambda c: any(a == 16 and b == 2 for _, _, a, b, _ in c["split_pairs"]),
    "S2 then S4": lambda c: any(a == 2 and b == 4 for _, _, a, b, _ in c["split_pairs"]),
    "S4 then whole tiles": lambda c: any(r.get("S") == 4 and _next_gemm_whole(c, i) for i, r in c["ops"].items()),
    "mid-ring phase 1": lambda c: all(mid_ring_phase1(c).values()),
    "war": lambda c: bool(c["war"]),
    "segment break": lambda c: len(c["segments"]) > 1,
    "multi-op segments": lambda c: any(n and n > 1 for n in c["segments"]),
}


def _next_gemm_whole(cov: dict, i: int) -> bool:
    later = sorted(j for j, r in cov["ops"].items() if j > i and "S" in r and r["segment"] == cov["ops"][i]["segment"])
    return bool(later) and cov["ops"][later[0]]["S"] == 1


# The Llama-3-8B layer at B 32 (hidden 4096, Hq 32, Hkv 8, D 128, inter 14336)
H8B, I8B, QKV8B = 4096, 14336, (32 + 2 * 8) * 128


def _layer(fmt):
    return (gemm("attn", "o", fmt, H8B, H8B), norm("o", "x1", H8B, res="res"), gemm("x1", "act", fmt, H8B, 2 * I8B, silu=True),
            gemm("act", "w2", fmt, I8B, H8B, bias=True), norm("w2", "x2", H8B, res="res"), gemm("x2", "qkv", fmt, H8B, QKV8B),
            rope("qkv", "q"))


def _ring(fmt, n):
    Ks = (384, 640, 896)
    return tuple(gemm(f"in{K}", f"r{i}", fmt, K, 240 * TILE_N) for i, K in zip(range(n), Ks * n))


CHAINS = [
    # imbalance: a 1-tile GEMM (4 contributors, 260 CTAs idle) -> norm with residual -> GEMM
    Chain("imbalance 1-tile gemm -> add_rmsnorm -> gemm int4 f16 b1", "f16", 1,
          (gemm("x", "h", "int4", 512, 128), norm("h", "hn", 128, res="res"), gemm("hn", "y", "int4", 128, 256, bias=True)),
          ("idle>250 then glue", "multi-op segments")),
    Chain("imbalance 1-tile gemm -> add_rmsnorm -> gemm int8 bf16 b17", "bf16", 17,
          (gemm("x", "h", "int8", 512, 128, bias=True), norm("h", "hn", 128, res="res"), gemm("hn", "y", "int8", 128, 384)),
          ("idle>250 then glue", "multi-op segments")),
    # imbalance: 3 whole tiles per CTA, then a GEMM consuming all 76800 features
    Chain("imbalance whole tiles x3 -> consumer int8 bf16 b16", "bf16", 16,
          (gemm("x", "h", "int8", 256, 76800), gemm("h", "y", "int8", 76800, 128, bias=True)),
          ("several tiles per CTA", "multi-op segments")),
    # split-K state: S 16 -> S 2 -> S 4 -> whole tiles on one workspace, each reading the previous output
    Chain("split-K S16 -> S2 -> S4 -> whole int8 f16 b33", "f16", 33,
          (gemm("x", "s1", "int8", 2048, 1024), gemm("s1", "s2", "int8", 1024, 12800, bias=True),
           gemm("s2", "s3", "int8", 12800, 128), gemm("s3", "y", "int8", 128, 512)),
          ("S16 then S2", "S2 then S4", "S4 then whole tiles", "multi-op segments")),
    Chain("split-K S16 -> S2 -> S4 -> whole int4 bf16 b64", "bf16", 64,
          (gemm("x", "s1", "int4", 2048, 1024, bias=True), gemm("s1", "s2", "int4", 1024, 12800),
           gemm("s2", "s3", "int4", 12800, 128), gemm("s3", "y", "int4", 128, 512, bias=True)),
          ("S16 then S2", "S2 then S4", "S4 then whole tiles", "multi-op segments")),
    # ring carry-over: 3 / 5 / 7 k-blocks per CTA (whole tiles), so op boundaries fall mid-ring with either phase
    Chain("ring carry-over 14 gemms int4 f16 b16", "f16", 16, _ring("int4", 14), ("mid-ring phase 1", "multi-op segments")),
    Chain("ring carry-over 12 gemms int8 bf16 b64", "bf16", 64, _ring("int8", 12), ("mid-ring phase 1", "multi-op segments")),
    # the Llama-3-8B layer between two attention calls
    Chain("layer Llama-3-8B int4 f16 b32", "f16", 32, _layer("int4"), ("multi-op segments",), Hq=32, Hkv=8),
    Chain("layer Llama-3-8B int8 bf16 b32", "bf16", 32, _layer("int8"), ("multi-op segments",), Hq=32, Hkv=8),
    # glue-led segments: the rope reads the page list written in the same launch
    Chain("glue-led table -> embedding -> norm -> gemm -> rope f16 b33", "f16", 33,
          (table("bid", "pl"), embed("ids", "e", 512), norm("e", "en", 512), gemm("en", "qkv", "int4", 512, 1536), rope("qkv", "q")),
          ("multi-op segments",)),
    Chain("glue-led table -> rope bf16 b17", "bf16", 17, (table("bid", "pl"), rope("qkv", "q")), ("multi-op segments",)),
    # WAR: the norm writes the first GEMM's input, the second GEMM writes the norm's input
    Chain("war gemm A->B, norm B->A, gemm A->B int4 bf16 b17", "bf16", 17,
          (gemm("A", "B", "int4", 1024, 1024), norm("B", "A", 1024, res="res"), gemm("A", "B", "int4", 1024, 1024, bias=True)),
          ("war", "multi-op segments")),
    Chain("war gemm A->B, norm B->A, gemm A->B int8 f16 b64", "f16", 64,
          (gemm("A", "B", "int8", 2048, 2048), norm("B", "A", 2048, res="res"), gemm("A", "B", "int8", 2048, 2048)),
          ("war", "multi-op segments")),
    # segment breaks
    Chain("break int4 -> int8 gemm f16 b33", "f16", 33,
          (gemm("x", "h", "int4", 1024, 2048), norm("h", "hn", 2048, res="res"), gemm("hn", "y", "int8", 2048, 1024)),
          ("segment break", "multi-op segments")),
    Chain("break int8g gemm and hidden-9216 norm mid-chain f16 b16", "f16", 16,
          (gemm("x", "a", "int4", 1024, 9216), norm("a", "an", 9216, res="res"), gemm("an", "b", "int8g", 9216, 1024),
           gemm("b", "c", "int4", 1024, 2048), norm("c", "y", 2048)),
          ("segment break", "multi-op segments")),
    Chain("break attention between rope and o gemm bf16 b17", "bf16", 17,
          (gemm("x", "qkv", "int4", 1024, 1536), rope("qkv", "q"), attn("q", "att"), gemm("att", "o", "int4", 1024, 1024),
           norm("o", "y", 1024, res="res")),
          ("segment break", "multi-op segments")),
]


def buffer_roles(chain: Chain) -> Dict[str, str]:
    """"in": read before any op writes it (seeded per input version; compared when an op writes it); "out": written first
    (NaN sentinel before every launch, compared). The K/V pool and a norm's residual count as read first."""
    roles: Dict[str, str] = {}
    for op in chain.ops:
        for b in op.reads():
            roles.setdefault(b, "in")
        for b in op.writes():
            roles.setdefault(b, "out")
    return roles


def written(chain: Chain) -> List[str]:
    seen: List[str] = []
    for op in chain.ops:
        for b in op.writes():
            if b not in seen:
                seen.append(b)
    return seen


def shapes(chain: Chain) -> Dict[str, Tuple[Tuple[int, ...], str]]:
    """name: (shape, "act" | "i32") of every buffer the chain names."""
    B, c = chain.B, chain
    s: Dict[str, Tuple[Tuple[int, ...], str]] = {}
    for op in chain.ops:
        if op.kind == "gemm":
            s[op.x] = ((B, op.K), "act")
            s[op.y] = ((B, op.N // 2 if op.silu else op.N), "act")
        elif op.kind == "norm":
            for b in (op.x, op.y) + ((op.res,) if op.res else ()):
                s[b] = ((B, op.hidden), "act")
        elif op.kind in ("rope", "attn"):
            s[op.x] = ((B, (c.Hq + 2 * c.Hkv) * c.D if op.kind == "rope" else c.Hq * c.D), "act")
            s[op.y] = ((B, c.Hq * c.D), "act")
            s["pool"] = ((B * c.M + 1, 2, c.Hkv, c.T, c.D), "act")
            s["pl"] = ((B, 1, 2, c.M), "i32")
            s["seq"] = ((B,), "i32")
        elif op.kind == "embed":
            s[op.x] = ((B,), "i32")
            s[op.y] = ((B, op.hidden), "act")
        elif op.kind == "table":
            s[op.x] = ((B, c.M), "i32")
            s[op.y] = ((B, 1, 2, c.M), "i32")
    return s


@dataclass
class Counts:
    """What a recording of a chain made: persistent-capable calls, separators, calls that are their own launch."""
    persistent: int = 0
    separators: int = 0
    plain: int = 0
