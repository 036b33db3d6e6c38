"""Model of the TP peer-collective region layout (csrc/peer_allreduce.cuh, b200_wo_gemm_rs) and exact numpy references of
the collectives, for running the peer kernels one rank at a time on one GPU.

Layout, restated from peer_strides in csrc/c_api.cu: a rank's region is [2 parities][2 areas][8 sources][LL slot], with
src = 2 * round_up(max_msg, 256) bytes per source, area = 8 * src, parity = 2 * area, and the call counter (uint32) at
2 * parity followed by the finishing-CTA ticket. A call with epoch e (= counter + 1) uses parity e & 1. Every payload word
travels as an 8-byte LL word {data32, e}; a 16-byte chunk is four of them (32 bytes).

Push sites (what rank `rank` writes into peer q's region, src = rank) and poll sites (what rank r reads from its own
region) are written out separately, each from its own lines of the kernels, so tests/test_peer_oracle.py can show that they
meet. Words are (byte offset, data32) pairs; the flag of every word is the call's epoch."""
import numpy as np

from oracle import oracle as orc

MAX_WORLD = 8
MAX_CTAS = 64
THREADS = 256
POISON_SUM = 0x7FFF7FFF      # a NaN in fp16 and in bf16 (both halves): a sum that reads it is NaN
POISON_ARGMAX = 0x7F800000   # as the value +inf (it wins), as the index 2139095040 (no vocabulary is that large)


def round_up(v, a):
    return (v + a - 1) // a * a


class Layout:
    def __init__(self, max_msg: int):
        self.max_msg = max_msg
        self.src = 2 * round_up(max_msg, 256)
        self.area = MAX_WORLD * self.src
        self.parity = 2 * self.area
        self.counter = 2 * self.parity              # uint32 call counter, then the ticket
        self.region_bytes = 2 * self.parity + MAX_CTAS * 4 + 256   # b200_peer_ar_region_bytes

    def base(self, epoch: int, area: int, src: int) -> int:
        """Byte offset of source `src`'s slot in `area` of the parity of `epoch`."""
        return (epoch & 1) * self.parity + area * self.area + src * self.src


def _ll(base, chunk_ids, words4):
    """Offsets and data of the LL words of 16-byte chunks: chunk c at slot chunk_ids[c] * 32 holds words4[c, 0..3] as four
    {data, flag} words, word k at +8k (push_chunk's two st_ll2)."""
    chunk_ids = np.asarray(chunk_ids, np.int64).reshape(-1)
    off = base + chunk_ids[:, None] * 32 + np.arange(4, dtype=np.int64)[None, :] * 8
    return off.reshape(-1), np.asarray(words4, np.uint32).reshape(-1)


def words_of(bits16) -> np.ndarray:
    """T bit patterns [..., 2m] (uint16) -> uint32 words [..., m] as the kernels see them (element 2i in the low half)."""
    b = np.ascontiguousarray(bits16, np.uint16)
    return b.view(np.uint32)


def merge(*parts):
    """Concatenate (offsets, data) pairs."""
    parts = [p for p in parts if len(p[0])]
    if not parts:
        return np.zeros(0, np.int64), np.zeros(0, np.uint32)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


# ---------------------------------------------------------------------------------------------- all-reduce
def allreduce_two_shot(n16: int, world: int, forced=None) -> bool:
    """The path b200_peer_allreduce takes: two-shot when B200_AR_TWOSHOT (`forced`; default world >= 3) asks for it and
    n16 % world == 0, one-shot otherwise."""
    want = (world >= 3) if forced is None else bool(int(forced))
    return want and n16 % world == 0


def allreduce_ctas(n16: int, world: int, two_shot: bool) -> int:
    c = -(-(n16 // world) // THREADS) if two_shot else -(-n16 // (2 * THREADS))
    return min(max(c, 1), MAX_CTAS)


def allreduce_pushes(lay: Layout, rank: int, world: int, epoch: int, mine_words, reduced_words, two_shot: bool):
    """{peer q: (offsets, data)} that rank `rank` writes into q's region. mine_words: this rank's input as uint32 [n16 * 4];
    reduced_words: the all-reduced result (the two-shot all-gather pushes this rank's slice of it)."""
    mine = np.asarray(mine_words, np.uint32).reshape(-1, 4)
    red = np.asarray(reduced_words, np.uint32).reshape(-1, 4)
    n16 = mine.shape[0]
    out = {}
    for q in range(world):
        if q == rank:
            continue
        if not two_shot:    # peer_allreduce_kernel: chunk i of my data -> area 0, slot [rank], chunk i
            out[q] = _ll(lay.base(epoch, 0, rank), np.arange(n16), mine)
        else:               # scatter: slice q of my data -> q's area 0; all-gather: my reduced slice -> q's area 1
            ns = n16 // world
            j = np.arange(ns)
            out[q] = merge(_ll(lay.base(epoch, 0, rank), j, mine[q * ns:(q + 1) * ns]),
                           _ll(lay.base(epoch, 1, rank), j, red[rank * ns:(rank + 1) * ns]))
    return out


def allreduce_polls(lay: Layout, rank: int, world: int, epoch: int, n16: int, two_shot: bool) -> np.ndarray:
    """Byte offsets of the LL words rank `rank` polls in its own region (poll_chunk's addresses, both 16-byte halves)."""
    offs = []
    for s in range(world):
        if s == rank:
            continue
        if not two_shot:
            offs.append(_ll(lay.base(epoch, 0, s), np.arange(n16), np.zeros((n16, 4)))[0])
        else:
            ns = n16 // world
            for area in (0, 1):
                offs.append(_ll(lay.base(epoch, area, s), np.arange(ns), np.zeros((ns, 4)))[0])
    return np.concatenate(offs) if offs else np.zeros(0, np.int64)


def sum_in_rank_order(contribs, is_bf16: bool, first=None) -> np.ndarray:
    """round_T of the fp32 sum 0 + c_0 + c_1 + ... + c_{W-1} (the kernels' acc2 chain), as T bits. contribs: [W, ...] uint16
    bit patterns. first: sum rank `first` first and the others after it in rank order (a mutant, for the tests)."""
    c = np.asarray(contribs, np.uint16)
    order = list(range(c.shape[0]))
    if first is not None:
        order = [first] + [q for q in order if q != first]
    acc = np.zeros(c.shape[1:], np.float32)
    for q in order:
        acc = acc + orc.from_bits(c[q], is_bf16).astype(np.float32)
    return orc.f64_to_bits(acc.astype(np.float64), is_bf16)


def crafted_order_input(world: int, n: int, is_bf16: bool, seed: int = 0) -> np.ndarray:
    """[W, n] T bits, N(0, 1) except element 0, whose fp32 sum depends on the order of the terms: c_0 = 2^15, c_1 = -2^15,
    every other rank 2^-10 (below half an fp32 ulp of 2^15). In rank order the big terms cancel first and the small ones
    survive; a rank >= 2 that adds its own term first loses it. (Ranks 0 and 1 add the same first two terms either way.)"""
    v = orc.round_t(np.random.default_rng(seed).standard_normal((world, n)), is_bf16)
    v[:, 0] = 2.0 ** -10
    v[0, 0], v[1, 0] = 2.0 ** 15, -2.0 ** 15
    return orc.f64_to_bits(v, is_bf16)


# ---------------------------------------------------------------------------------------------- all-reduce + norm
def norm_slots(rows: int, hidden: int, world: int):
    """(C, Cs): 16-byte chunks per row and per owner's slice."""
    C = hidden // 8
    return C, C // world


def norm_pushes(lay: Layout, rank: int, world: int, epoch: int, mine_bits, reduced_bits, pushed: bool = False):
    """{peer q: (offsets, data)} of peer_allreduce_norm_kernel on rank `rank`: phase 1 (skipped when `pushed`) sends chunk c
    of each row to its owner c // Cs at slot row * Cs + (c - owner * Cs) of area 0; phase 2 sends the rank's reduced slice
    (chunks rank * Cs .. + Cs of each row) to every peer's area 1 at slot row * Cs + cs."""
    mine = words_of(mine_bits)
    rows = mine.shape[0]
    C, Cs = norm_slots(rows, mine.shape[1] * 2, world)
    mine = mine.reshape(rows, C, 4)
    red = words_of(reduced_bits).reshape(rows, C, 4)
    row = np.arange(rows)[:, None]
    cs = np.arange(Cs)[None, :]
    out = {}
    for q in range(world):
        if q == rank:
            continue
        parts = []
        if not pushed:
            parts.append(_ll(lay.base(epoch, 0, rank), row * Cs + cs, mine[:, q * Cs:(q + 1) * Cs]))
        parts.append(_ll(lay.base(epoch, 1, rank), row * Cs + cs, red[:, rank * Cs:(rank + 1) * Cs]))
        out[q] = merge(*parts)
    return out


def norm_polls(lay: Layout, rank: int, world: int, epoch: int, rows: int, hidden: int) -> np.ndarray:
    C, Cs = norm_slots(rows, hidden, world)
    offs = []
    for s in range(world):
        if s == rank:
            continue
        # phase 2 polls slot row * Cs + cs of source s in area 0; phase 3 polls, for chunk c owned by s, slot
        # row * Cs + (c - s * Cs) of source s in area 1
        ids = np.arange(rows)[:, None] * Cs + np.arange(Cs)[None, :]
        c = np.arange(C)
        owner = c // Cs
        ids3 = np.arange(rows)[:, None] * Cs + (c[owner == s] - s * Cs)[None, :]
        offs.append(_ll(lay.base(epoch, 0, s), ids, np.zeros(ids.shape + (4,)))[0])
        offs.append(_ll(lay.base(epoch, 1, s), ids3, np.zeros(ids3.shape + (4,)))[0])
    return np.concatenate(offs) if offs else np.zeros(0, np.int64)


def norm_chain(hidden: int) -> int:
    """The longest fp32 add chain of peer_allreduce_norm_kernel's sum of squares: 8 fmaf per 16-byte chunk, ceil(C / 256)
    chunks per thread, then 5 butterfly levels and the sum of the 8 warp partials."""
    return 8 * (-(-(hidden // 8) // THREADS)) + 5 + 8


def allreduce_norm_ref(contribs, residual_bits, gamma_bits, eps, is_bf16: bool, round_reduced: bool = True):
    """The fused kernel's contract. contribs [W, rows, hidden] uint16; residual / gamma T bits.
    Returns (reduced bits, stored residual bits, y float64, A): reduced = round_T(fp32 rank-order sum); x = the fp32 sum
    float(reduced) + float(residual), unrounded; stored residual = round_T(x) (inf where it overflows); y = the float64
    RMSNorm of x (oracle.rmsnorm_np) with A its term size for oracle.norm_error_budget. round_reduced=False: the mutant that
    adds the fp32 sum without rounding it to T first."""
    red = sum_in_rank_order(contribs, is_bf16)
    if round_reduced:
        a = orc.from_bits(red, is_bf16).astype(np.float64)
    else:
        acc = np.zeros(np.asarray(contribs).shape[1:], np.float32)
        for c in contribs:
            acc = acc + orc.from_bits(c, is_bf16).astype(np.float32)
        a = acc.astype(np.float64)
    r = orc.from_bits(residual_bits, is_bf16).astype(np.float64)
    s = a + r
    bb = s - a
    assert np.all((a - (s - bb)) + (r - bb) == 0.0), "reduced + residual is not exact in float64"
    x = s.astype(np.float32).astype(np.float64)          # the one fp32 rounding of the kernel's add
    stored = orc.f64_to_bits(x, is_bf16)
    y, _, A = orc.rmsnorm_np(x, None, orc.from_bits(gamma_bits, is_bf16).astype(np.float64), eps)
    return red, stored, y, A


# ---------------------------------------------------------------------------------------------- reduce-scatter GEMM
def rs_gemm_pushes(lay: Layout, rank: int, world: int, epoch: int, y_bits):
    """{peer q: (offsets, data)} of b200_wo_gemm_rs on rank `rank` (rs_lane / rs_emit): the pair of columns (n, n + 1), n even,
    of row b goes, when its owner o = (n / 8) / Cs is not this rank, to o's area 0, slot [rank], at
    (c - o * Cs) * 32 + ((n & 7) >> 1) * 8 + b * Cs * 32 with c = n / 8. y_bits: the plain GEMM's output [B, N] (uint16)."""
    words = words_of(y_bits)                            # [B, N / 2]: word n / 2 holds columns n, n + 1
    B, half = words.shape
    N = 2 * half
    Cs = N // 8 // world
    n = np.arange(0, N, 2)
    c = n >> 3
    owner = c // Cs
    out = {}
    for q in range(world):
        if q == rank:
            continue
        sel = owner == q
        col = ((c[sel] - q * Cs) * 32 + ((n[sel] & 7) >> 1) * 8)[None, :]
        off = lay.base(epoch, 0, rank) + col + np.arange(B, dtype=np.int64)[:, None] * (Cs * 32)
        out[q] = (off.reshape(-1).astype(np.int64), words[:, sel].reshape(-1))
    return out


def owned_columns(N: int, world: int, rank: int) -> slice:
    Cs = N // 8 // world
    return slice(rank * Cs * 8, (rank + 1) * Cs * 8)


# ---------------------------------------------------------------------------------------------- argmax
def argmax_np(logits) -> np.ndarray:
    """b200_argmax's contract on float rows: the largest value, lowest index on ties; NaN never wins; a row of -inf gives
    index 0 (the lowest among equals); a row with nothing but NaN gives 0x7fffffff (no candidate)."""
    v = np.asarray(logits, np.float64)
    out = np.full(v.shape[0], 0x7FFFFFFF, np.int64)
    for i, row in enumerate(v):
        ok = ~np.isnan(row)
        if ok.any():
            m = row[ok].max()
            out[i] = int(np.flatnonzero(ok & (row == m))[0])
    return out


def argmax_local(logits, rank: int, vocab_local: int, vocab_total: int):
    """(value as fp32 bits, global index) per row that rank `rank` computes over its shard: columns rank * vocab_local + i
    below vocab_total only, -inf / 0x7fffffff when nothing qualifies (b200_argmax's rule on the shard)."""
    v = np.asarray(logits, np.float64)[:, :max(0, min(vocab_local, vocab_total - rank * vocab_local))]
    val = np.full(v.shape[0], -np.inf)
    idx = np.full(v.shape[0], 0x7FFFFFFF, np.int64)
    if v.shape[1]:
        loc = argmax_np(v)
        has = loc != 0x7FFFFFFF
        val[has] = v[np.flatnonzero(has), loc[has]]
        idx[has] = loc[has] + rank * vocab_local
    return val.astype(np.float32).view(np.uint32), idx.astype(np.uint32)


def argmax_pushes(lay: Layout, rank: int, world: int, epoch: int, val_bits, idx):
    """{peer q: (offsets, data)}: row r's pair goes to q's area 0, slot [rank], at row * 16: {value, e} then {index, e}."""
    rows = len(idx)
    off = lay.base(epoch, 0, rank) + np.arange(rows, dtype=np.int64)[:, None] * 16 + np.array([0, 8])[None, :]
    data = np.stack([np.asarray(val_bits, np.uint32), np.asarray(idx, np.uint32)], 1)
    return {q: (off.reshape(-1), data.reshape(-1)) for q in range(world) if q != rank}


def argmax_polls(lay: Layout, rank: int, world: int, epoch: int, rows: int) -> np.ndarray:
    offs = [lay.base(epoch, 0, s) + np.arange(rows, dtype=np.int64)[:, None] * 16 + np.array([0, 8])[None, :]
            for s in range(world) if s != rank]
    return np.concatenate([o.reshape(-1) for o in offs]) if offs else np.zeros(0, np.int64)


def polled_by(pushes_of_peers, rank: int):
    """The words rank `rank` finds in its region: what every peer pushed to it. pushes_of_peers: {src: {dst: (off, data)}}."""
    return merge(*[p[rank] for s, p in pushes_of_peers.items() if s != rank])
