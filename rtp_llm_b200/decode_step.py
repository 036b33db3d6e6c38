"""One decode step of a dense Llama/Qwen-style stack on the H100 hot path (synthetic weights, synthetic page tables).

This is the measurement harness of SURVEY.md section 8(d): per layer
    add_rmsnorm -> qkv GEMM -> [QK-norm +] rope + KV append -> paged decode attention -> o GEMM -> [TP all-reduce]
    -> add_rmsnorm -> w13 GEMM -> SiLU*mul -> w2 GEMM -> [TP all-reduce]
then final norm -> lm_head (fp16 weights) -> greedy argmax, all on one stream under one CUDA graph.
It mirrors the call order of the reference's Python model graph (model_desc/qwen3.py:57-138,
modules/hybrid/causal_attention.py:75-93, modules/hybrid/dense_mlp.py:95-106, PyWrappedModel.cc:938-1060) but owns none
of its engine: scheduler, cache manager and sampler policy stay the reference's.
"""
from __future__ import annotations

import dataclasses
import math
import os
from typing import Dict, List, Mapping, Optional, Sequence, Union

import torch

from . import ops, rope
from ._lib import B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT8, B200_FMT_INT8G
from .attention import beam_rows_fit
from .rope import LLAMA3, RopeSpec


@dataclasses.dataclass
class ModelConfig:
    name: str
    hidden: int
    layers: int
    head_num: int
    kv_head_num: int
    head_dim: int
    inter: int
    vocab: int
    rope_base: float = 500000.0
    eps: float = 1e-5
    quant: str = "int4"          # "f16" | "int8" (per column) | "int4" (group 128) | "int8g" (8-bit group 128)
    tokens_per_block: int = 64   # KVCacheConfig.seq_size_per_block default (ConfigModules.h:174)
    # None: plain Base rotation at rope_base. A rope config replaces rope_base; the step appends through rope.rope_append,
    # which runs b200_rope_append(_multi) for a plain Base config and b200_rope_append_ex(_multi) for every other one, with
    # the cos/sin table for Base and Yarn (rope.py).
    rope: Optional[RopeSpec] = None
    # Qwen3's QK-norm: every layer carries q_norm / k_norm gammas [head_dim], and each q and k head is RMS-normalised (eps) before
    # the rotation, inside the rope launch (rope.rope_append(qk_norm=...) -> b200_qk_norm_rope_append(_ex)).
    qk_norm: bool = False


LLAMA3_8B = ModelConfig("Llama-3-8B", 4096, 32, 32, 8, 128, 14336, 128256)
# Llama-3.1 / 3.2 / 3.3: Llama3 frequency scaling (factor 8, low / high frequency factor 1 / 4, original max positions 8192)
LLAMA31_8B = ModelConfig("Llama-3.1-8B", 4096, 32, 32, 8, 128, 14336, 128256,
                         rope=RopeSpec(style=LLAMA3, dim=128, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192))
QWEN2_72B = ModelConfig("Qwen2-72B", 8192, 80, 64, 8, 128, 29696, 152064, rope_base=1000000.0, eps=1e-6)  # GPTQ-padded inter
TINY = ModelConfig("tiny", 512, 2, 4, 2, 128, 512, 1024, tokens_per_block=16)
QWEN3_8B = ModelConfig("Qwen3-8B", 4096, 36, 32, 8, 128, 12288, 151936, rope_base=1000000.0, eps=1e-6, qk_norm=True)
# Hq * D = 8192 != hidden 5120: the o projection is not square
QWEN3_32B = ModelConfig("Qwen3-32B", 5120, 64, 64, 8, 128, 25600, 151936, rope_base=1000000.0, eps=1e-6, qk_norm=True)
# the tests' Qwen3: QK-norm, and Hq * D = 1024 != hidden 512 as in Qwen3-32B
TINY_QWEN3 = ModelConfig("tiny-qwen3", 512, 2, 8, 2, 128, 512, 1024, rope_base=1000000.0, eps=1e-6, tokens_per_block=16,
                         qk_norm=True)


@dataclasses.dataclass
class SamplingParams:
    """Per-request sampling parameters of DecodeStep's sampling mode: each field is one value for every request or a sequence of
    one value per request, with b200_sample's meaning (top_k <= 0 and top_p >= 1: no limit; repetition 1, presence 0 and
    frequency 0: off; min_p in [0, 1], 0: off). seed fixes the step's uniforms (sampling_uniforms)."""
    temperature: Union[float, Sequence[float]] = 1.0
    top_k: Union[int, Sequence[int]] = 0
    top_p: Union[float, Sequence[float]] = 1.0
    repetition: Union[float, Sequence[float]] = 1.0
    presence: Union[float, Sequence[float]] = 0.0
    frequency: Union[float, Sequence[float]] = 0.0
    seed: int = 0
    min_p: Union[float, Sequence[float]] = 0.0

    def has_penalties(self) -> bool:
        return any(any(float(v) != off for v in (x if isinstance(x, (list, tuple)) else [x]))
                   for x, off in ((self.repetition, 1.0), (self.presence, 0.0), (self.frequency, 0.0)))

    def has_min_p(self) -> bool:
        return any(float(v) != 0.0 for v in (self.min_p if isinstance(self.min_p, (list, tuple)) else [self.min_p]))


_U32 = 0xFFFFFFFF


def _mix32(x: torch.Tensor, tmp: torch.Tensor) -> None:
    """A 32-bit integer hash, in place on int64 values in [0, 2^32): xor-shift / multiply rounds whose multipliers stay below
    2^31, so no product leaves int64. tmp: scratch of x's shape."""
    for shift, mul in ((16, 0x7FEB352D), (15, 0x2C1B3C6D), (16, 0)):
        torch.bitwise_right_shift(x, shift, out=tmp)
        x.bitwise_xor_(tmp)
        if mul:
            x.mul_(mul).bitwise_and_(_U32)


class _Uniforms:
    """n uniforms in [0, 1) per step, a pure function of (seed, step, i): u = (h(h(h(seed + 0x9E3779B9) ^ step) ^ i) >> 8) / 2^24
    with h = _mix32 (all mod 2^32) and
    `step` an int64 [1] tensor. Torch ops into static buffers only, so a CUDA graph replays them and each replay draws from the
    step counter it finds on the device."""

    def __init__(self, seed: int, n: int, device):
        self.key = torch.tensor([(seed + 0x9E3779B9) & _U32], dtype=torch.int64, device=device)
        self.k1, self.t1 = torch.empty_like(self.key), torch.empty_like(self.key)
        _mix32(self.key, self.t1)
        self.idx = torch.arange(n, dtype=torch.int64, device=device)
        self.x, self.t = torch.empty_like(self.idx), torch.empty_like(self.idx)

    def draw(self, step: torch.Tensor, out: torch.Tensor) -> None:
        torch.bitwise_xor(self.key, step, out=self.k1)
        _mix32(self.k1, self.t1)
        torch.bitwise_xor(self.k1, self.idx, out=self.x)
        _mix32(self.x, self.t)
        self.x.bitwise_right_shift_(8)
        out.copy_(self.x)
        out.mul_(1.0 / (1 << 24))


def sampling_uniforms(seed: int, step: int, n: int) -> torch.Tensor:
    """The n uniforms (fp32, CPU) the sampling mode draws at `step` (0 = the first step since upload_inputs()): the first
    B * q_len go to b200_sample's rows, at q_len > 1 the next B * q_len to b200_spec_verify."""
    u = _Uniforms(seed, n, "cpu")
    out = torch.empty(n, dtype=torch.float32)
    u.draw(torch.tensor([step], dtype=torch.int64), out)
    return out


def _fmt(q: str) -> int:
    return {"f16": B200_FMT_F16, "int8": B200_FMT_INT8, "int4": B200_FMT_INT4, "int8g": B200_FMT_INT8G}[q]


def weight_bytes(cfg: ModelConfig, K: int, N: int) -> float:
    """Algorithmic HBM bytes of one weight (SURVEY 8d: int4 = E/2 + (E/128)*4, int8 = E + 2N, f16 = 2E)."""
    E = K * N
    if cfg.quant == "int4":
        return E / 2 + E / 128 * 4
    if cfg.quant == "int8":
        return E + 2 * N
    if cfg.quant == "int8g":
        return E + E / 128 * 4
    return 2 * E


class DecodeStep:
    """Synthetic decode step. tp_size > 1 shards exactly as the reference's TP split (utils/model_weight.py:1489-1580):
    qkv / w13 column-parallel, o / w2 row-parallel + all-reduce, lm_head vocab-parallel + all-gather.

    act_order=True (TP 1, quant int4 / int8g): every quantised weight is a GPTQ act-order weight with its rows sorted by g_idx,
    from seeded random row orders. qkv, o and w13 carry theirs in the blob, and x is gathered (b200_permute_cols) into a static
    buffer before each of them; w2's order is folded into w13's output columns, as B200Loader.layer does. A row-parallel o
    shard would mix groups of every rank, so TP > 1 is rejected.

    q_len > 1 (TP 1, op by op or under a CUDA graph; not in a decode program): a verification step of speculative tokens. Each
    sequence feeds q_len tokens, ids_h [B, q_len] = the last accepted token and q_len - 1 drafts, at positions seq_lens_h[b] + j.
    Every op runs on the B * q_len rows (rope_append / paged_decode_attn_multi for the attention), argmax picks each row's
    token, and spec_verify (greedy) checks the drafts against them: out_tokens [B, q_len], accepted [B].

    beam_width W > 1 (TP 1, q_len 1, op by op or under a CUDA graph; not in a decode program): beam search over `batch` requests.
    Each beam is a sequence of its own, so every op runs on B * W rows, row b * W + i = beam i of request b, with its own
    page-table row. The prompt (ctx - max_new_tokens tokens already cached) shares its full pages among a request's W beams;
    from the prompt's last, partial page onward every beam owns private pages. The step ends in ban_repeat_ngram (when
    no_repeat_ngram > 0) and beam_search_step instead of argmax, then forks in place with static buffers: cum_log_probs takes
    next_cum, the token history rows are gathered by next_parent and the new token appended, new beam j takes its parent's
    page-table entries for the full pages, and the parent's partial last page is copied into j's own page (every source page
    gathered into scratch first, then scattered, since a beam can be a parent and a child in the same step). Then the ids
    become next_token and the lengths grow by one: the next call runs the next step. upload_inputs() restarts from the prompt;
    a step past max_new_tokens since then raises ValueError (the page-table rows end there), in run() and in replay().
    The attention reads that shared prompt once per request: when attention.beam_rows_fit holds (group * W <= 64 query rows and
    at least 128 (request, kv head) pairs, from where the kernel was measured to win) the layers call paged_decode_attn_beam with shared_lens [B] = the prompt's full pages * tokens_per_block, a static buffer
    that upload_inputs() refreshes (the prompt is fixed between two uploads, so a graph replays it); a wider search runs
    paged_decode_attn on the B * W rows. The invariant this rests on: the fork gives a new beam its parent's page-table entries
    for every page the step has filled, and all parents descend from the prompt's beams, so at every step the W page-table rows
    of a request are equal over the first shared_lens[b] / tokens_per_block pages.
    The device state: beam_cum [B, W], hist [B*W, ctx] / hist_len [B*W], beam_out (the beam_search_step outputs).
    With eos_id, finished hypotheses are kept on the device: beam_search_step runs with that EOS (the next beams skip it), then
    beam_hypotheses_update moves the EOS candidates among the first W ranks into each request's set (hyp_state, up to W paths
    of max_new_tokens; history from hist[:, 1:], hist[:, 0] being the input token) before the fork. length_penalty (alpha,
    score = cum / len^alpha) and early_stopping (False, True or "never") take one value for every request or one per request.
    done [B] (int32, device) is set when a request's set is done; its beams keep computing (the graph is static) but its
    hypotheses stay as they are. beam_results(n) returns the n best per request, the live beams merged in for requests that are
    not done. upload_inputs() empties the sets and done. With eos_id None the step is the beam step without EOS.

    sampling=SamplingParams (TP 1, beam_width 1, batch * q_len <= 128, op by op or under a CUDA graph; not in a decode program):
    sampled decoding. The per-request parameters sit in static device buffers; after the lm_head the step copies the logits to a
    static fp32 buffer (samp_logits: b200_sample works in place and leaves the probabilities there), runs ban_repeat_ngram when
    no_repeat_ngram > 0, then b200_sample with the row's token history for the penalties. Its uniforms (one per row, `uniform`)
    are drawn on the device inside the step from (seed, step since upload_inputs()), see sampling_uniforms, so every graph
    replay draws new ones. With logprobs = n >= 0, b200_token_logprobs then scores the raw lm_head output: the drawn token's
    log-prob and the top n (lp_out); with logprobs None it does not run.
    At q_len 1 the step advances as the beam mode does: cum_log_probs += log(token_prob) (the reference's rule), the token
    joins the history, ids become the drawn tokens and the lengths grow by one; upload_inputs() restarts from the prompt and a
    step past max_new_tokens raises ValueError.
    At q_len > 1 it verifies drafts by sampling: b200_sample runs over the B * q_len rows with probs_out into target_probs
    [B, q_len, V], then spec_verify in sampling mode with deterministic drafts (draft_probs None) and its own uniforms [B, q_len].
    Like the greedy verification step it does not advance. Penalties and the n-gram ban are rejected there: row j's history
    would have to hold drafts 0..j-1. SamplingParams.min_p runs b200_sample with a min_p buffer when some value is not 0, and
    without one (today's kernel call) when every value is 0.

    tree=parents (q_len = n >= 2 nodes, greedy or sampled verification; TP 1, op by op or under a CUDA graph, with or without
    PDL; not in a decode program): verification of a speculative token tree. parents is one list of n entries for every request
    or one per request (parents[0] = -1, node j under parents[j] < j); set_tree() replaces it between replays. ids_h [B, n] holds
    the root (the last accepted token) and node j's draft token in column j. Node j's K/V go to slot seq + j and it is rotated at
    position seq + depth(j): the positions are formed on the device from static parent / depth buffers and passed to
    rope.rope_append as position_ids, so by the seams' rule even a plain Base config runs the _ex rope kernels there. The layers
    call paged_decode_attn_tree; the ending is argmax (or b200_sample with probs_out) and spec_verify_tree, then one
    kv_compact_path over every layer moves the accepted path's K/V to slots seq .. seq + accepted. Like the chain step it does
    not advance; out_tokens [B, n], accepted [B] and accepted_path [B, n] hold the result, with one launch more than the chain
    step (the compaction). Constraints apply per row (row j carries node j's mask); penalties and the n-gram ban are rejected
    as for sampled chain verification.

    token_bitmask=True and / or logit_bias_capacity=n > 0 (TP 1, every mode): constrained decoding. Static device buffers,
    filled by set_constraints() from pinned host twins, hold one grammar bitmask row per logits row (int32 [R, ceil(V / 32)],
    xgrammar's layout) and a logit-bias CSR of up to n entries; a graph replay applies what was set last, and upload_inputs()
    resets them to unconstrained (all-ones mask, no bias entries). b200_constrain_logits runs once per step where the ending
    reads the logits: on self.logits before argmax (greedy and greedy verification; row j of a verification step carries the
    mask of position j), on samp_logits after the fp32 copy and before the n-gram ban and b200_sample (sampling and sampled
    verification), on self.logits before the n-gram ban and beam_search_step (beam: one row per beam, before the
    log-softmax). The log-probs keep scoring the raw lm_head output. Without these options the step's launches are unchanged."""

    def __init__(self, cfg: ModelConfig, batch: int, ctx: int, device: torch.device, tp_rank: int = 0, tp_size: int = 1,
                 dtype=torch.float16, seed: int = 0, keep_reference: bool = False, ragged: bool = False,
                 pdl: bool = False, comm=None, fuse_silu: bool = True, fuse_ar_norm: bool = True, fuse_rope: Optional[bool] = None,
                 fuse_gemm_rs: Optional[bool] = None, act_order: bool = False, q_len: int = 1, beam_width: int = 1,
                 no_repeat_ngram: int = 0, max_new_tokens: int = 16, sampling: Optional[SamplingParams] = None,
                 logprobs: Optional[int] = None, eos_id: Optional[int] = None,
                 length_penalty: Union[float, Sequence[float]] = 1.0,
                 early_stopping: Union[bool, str, Sequence[Union[bool, str]]] = False,
                 token_bitmask: bool = False, logit_bias_capacity: int = 0, tree=None):
        assert cfg.head_num % tp_size == 0 and cfg.inter % tp_size == 0
        if logit_bias_capacity < 0:
            raise ValueError(f"logit_bias_capacity must be >= 0 (got {logit_bias_capacity})")
        if (token_bitmask or logit_bias_capacity) and tp_size != 1:
            raise ValueError(f"token_bitmask / logit_bias need tp_size 1 (got tp_size {tp_size}): the vocabulary-parallel argmax "
                             "would need a mask sharded by vocabulary")
        if sampling is not None:
            mp = sampling.min_p if isinstance(sampling.min_p, (list, tuple)) else [sampling.min_p]
            if not all(0.0 <= float(v) <= 1.0 for v in mp):
                raise ValueError(f"sampling: min_p must be in [0, 1] (got {sampling.min_p})")
        if q_len < 1:
            raise ValueError(f"q_len must be >= 1 (got {q_len})")
        if q_len > 1 and (batch * q_len > 128 or tp_size != 1):
            raise ValueError(f"a verification step (q_len {q_len}) needs batch * q_len <= 128 (the GEMM row limit) and tp_size 1 "
                             f"(got batch {batch}, tp_size {tp_size})")
        if tree is not None and q_len < 2:
            raise ValueError(f"a token-tree step needs q_len >= 2 nodes (got q_len {q_len})")
        if not 1 <= beam_width <= 32:
            raise ValueError(f"beam_width must be in 1..32 (got {beam_width})")
        if beam_width > 1 and (batch * beam_width > 128 or tp_size != 1 or q_len != 1):
            raise ValueError(f"beam search (beam_width {beam_width}) needs batch * beam_width <= 128 (the GEMM row limit), tp_size 1 "
                             f"and q_len 1 (got batch {batch}, tp_size {tp_size}, q_len {q_len})")
        if sampling is not None:
            if tp_size != 1 or beam_width != 1 or batch * q_len > 128:
                raise ValueError(f"sampling needs tp_size 1, beam_width 1 and batch * q_len <= 128 (the GEMM row limit) (got tp_size "
                                 f"{tp_size}, beam_width {beam_width}, batch {batch}, q_len {q_len})")
            if q_len > 1 and (sampling.has_penalties() or no_repeat_ngram != 0):
                raise ValueError("sampled verification (q_len > 1) takes no penalties and no n-gram ban: row j's history would "
                                 "have to hold drafts 0..j-1")
            if logprobs is not None and not 0 <= logprobs <= ops.LOGPROB_MAX_TOP_N:
                raise ValueError(f"logprobs must be in 0..{ops.LOGPROB_MAX_TOP_N} (got {logprobs})")
        elif logprobs is not None:
            raise ValueError("logprobs needs the sampling mode (sampling=SamplingParams(...))")
        self.samp = sampling
        self.logprobs = logprobs
        self.sample_advances = sampling is not None and q_len == 1
        if (beam_width > 1 or self.sample_advances) and not 1 <= max_new_tokens < ctx:
            raise ValueError(f"max_new_tokens must be in 1..ctx-1 (got {max_new_tokens}, ctx {ctx})")
        if no_repeat_ngram != 0 and beam_width == 1 and sampling is None:
            raise ValueError(f"no_repeat_ngram {no_repeat_ngram} needs beam search (beam_width > 1); the greedy step has no ban")
        self.W, self.ngram, self.max_new_tokens = beam_width, no_repeat_ngram, max_new_tokens
        if eos_id is not None:
            if beam_width == 1 or not 0 <= eos_id < cfg.vocab:
                raise ValueError(f"eos_id needs beam search (beam_width > 1) and must be in 0..vocab-1 (got eos_id {eos_id}, "
                                 f"beam_width {beam_width})")

            def per_request(v, name):
                vals = list(v) if isinstance(v, (list, tuple)) else [v] * batch
                if len(vals) != batch:
                    raise ValueError(f"{name}: {len(vals)} values for {batch} requests")
                return vals
            alphas = [float(a) for a in per_request(length_penalty, "length_penalty")]
            modes = per_request(early_stopping, "early_stopping")
            for m in modes:
                if m not in (False, True, "never"):
                    raise ValueError(f"early_stopping must be False, True or \"never\" (got {m!r})")
            modes = [2 if m == "never" else int(bool(m)) for m in modes]
        self.eos_id = eos_id
        self.beam_steps = 0                             # beam / sampled steps run since the prompt (upload_inputs)
        self.requests = batch
        batch = batch * beam_width                      # sequences (page-table rows) of the step
        self.q_len = q_len
        R = batch * q_len                               # token rows of the step
        if act_order and (tp_size != 1 or cfg.quant not in ("int4", "int8g")):
            raise ValueError(f"act_order needs tp_size 1 and quant int4 / int8g (got tp_size {tp_size}, quant {cfg.quant})")
        self.act_order = act_order
        self.cfg, self.B, self.ctx, self.dev, self.dtype = cfg, batch, ctx, device, dtype
        self.tp_rank, self.tp_size, self.comm, self.pdl = tp_rank, tp_size, comm, pdl
        self.Hq = cfg.head_num // tp_size
        self.Hkv = max(cfg.kv_head_num // tp_size, 1)   # kv heads replicated when Hkv < tp (MHAKVCacheSpec.h:46-51)
        self.D = cfg.head_dim
        self.inter = cfg.inter // tp_size
        assert (self.inter % 128 == 0) and (self.Hq * self.D) % 128 == 0, "row-parallel K must be a multiple of 128"
        self.vocab = (cfg.vocab + tp_size - 1) // tp_size
        self.vocab = (self.vocab + 7) // 8 * 8          # sp_0_pad8
        T = cfg.tokens_per_block
        self.M = (ctx + T - 1) // T
        self.ref: Dict[str, list] = {} if keep_reference else None
        self.fuse_silu = fuse_silu and self.inter % 64 == 0
        self.fuse_ar_norm = fuse_ar_norm
        # row-parallel GEMM + reduce-scatter in one kernel (b200_wo_gemm_rs), then gather + residual + norm (b200_peer_gather_norm):
        # only with the peer communicator and the fused all-reduce+norm; B200_FUSE_GEMM_RS=0 turns it off (A/B runs)
        if fuse_gemm_rs is None:
            fuse_gemm_rs = os.environ.get("B200_FUSE_GEMM_RS", "1") == "1"
        self.fuse_gemm_rs = (bool(fuse_gemm_rs) and fuse_ar_norm and tp_size > 1 and hasattr(comm, "gemm_rs")
                             and comm.gemm_rs_supported(batch, cfg.hidden))
        # RoPE + K/V append inside the attention kernel (b200_paged_decode_attn_rope): bit-identical, one launch less per layer,
        # but under PDL the stand-alone rope kernel hides behind its neighbours while the fused prologue sits on the attention
        # kernel's critical path.
        # Default off; B200_FUSE_ROPE=1 or fuse_rope=True turns it on.
        if fuse_rope is None:
            fuse_rope = os.environ.get("B200_FUSE_ROPE", "0") == "1"
        self.rope_spec = RopeSpec(dim=self.D, base=cfg.rope_base) if cfg.rope is None else rope.spec_of(cfg.rope, self.D)
        # the fused rope appends one token with plain Base rotation, and does not normalise q / k
        self.fuse_rope = (bool(fuse_rope) and cfg.head_dim == 128 and q_len == 1 and rope.is_plain_base(self.rope_spec, self.D)
                          and not cfg.qk_norm)
        g = torch.Generator(device="cpu").manual_seed(seed * 1000 + 17)
        H = cfg.hidden

        def pack_ref(refw, gate_up_inter: int = 0, perm=None, col_perm=None):
            """Reference-layout tuple -> kernel layout. gate_up_inter > 0: a [K, 2I] gate|up weight whose columns are
            first interleaved per 64 outputs so the GEMM epilogue can apply SiLU(gate)*up (ops.interleave_gate_up).
            perm: act-order row order carried by the blob; col_perm: w2's row order folded into a gate|up weight's columns."""
            fmt, w, s, zs = refw
            gi = gate_up_inter
            if fmt in ("int4", "int8g"):
                w, s, zs = w.to(device), s.to(device), zs.to(device)
                if col_perm is not None:
                    order = torch.cat([col_perm, col_perm + s.shape[1] // 2])
                    w = ops.permute_columns(w, order, packed_int4=fmt == "int4")
                    s, zs = ops.permute_columns(s, order), ops.permute_columns(zs, order)
                if gi:
                    w, s, zs = (ops.interleave_gate_up(w, gi, packed_int4=fmt == "int4"), ops.interleave_gate_up(s, gi),
                                ops.interleave_gate_up(zs, gi))
                return (ops.pack_w4 if fmt == "int4" else ops.pack_w8g)(w, s, zs, perm=perm)
            if fmt == "int8":
                w, s = w.to(device), s.to(device)
                if gi:
                    w, s = ops.interleave_gate_up(w, gi), ops.interleave_gate_up(s, gi)
                return ops.pack_w8(w, s)
            w = w.to(device)
            if gi:
                w = ops.interleave_gate_up(w, gi)
            return ops.pack_f16(w)

        def make_weight(K: int, N: int, gen_seed: int, quant: Optional[str] = None, gate_up_inter: int = 0, perm=None,
                        col_perm=None):
            quant = quant or cfg.quant
            gg = torch.Generator(device=device).manual_seed(gen_seed)
            if quant == "int4":
                qp = torch.randint(0, 256, (K, N // 2), generator=gg, device=device, dtype=torch.uint8)
                s = (torch.randn(K // 128, N, generator=gg, device=device).abs() * 0.01 + 1e-3).to(dtype)
                z = torch.randint(0, 16, (K // 128, N), generator=gg, device=device)
                zs = ((8 - z).to(dtype) * s).to(dtype)
                refw = ("int4", qp, s, zs)
            elif quant == "int8g":
                q8 = torch.randint(-128, 128, (K, N), generator=gg, device=device, dtype=torch.int8)
                s = (torch.randn(K // 128, N, generator=gg, device=device).abs() * 6e-4 + 6e-5).to(dtype)
                z = torch.randint(0, 256, (K // 128, N), generator=gg, device=device)
                zs = ((128 - z).to(dtype) * s).to(dtype)
                refw = ("int8g", q8, s, zs)
            elif quant == "int8":
                q8 = torch.randint(-128, 128, (K, N), generator=gg, device=device, dtype=torch.int8)
                s = (torch.randn(N, generator=gg, device=device).abs() * 2e-4 + 1e-5).to(dtype)
                refw = ("int8", q8, s, None)
            else:
                wkn = (torch.randn(K, N, generator=gg, device=device) * 0.02).to(dtype)
                refw = ("f16", wkn, None, None)
            w = pack_ref(refw, gate_up_inter, perm, col_perm)
            return w, (tuple(t.cpu() if torch.is_tensor(t) else t for t in refw) if keep_reference else None)

        self.layers: List[dict] = []
        qkv_n = (self.Hq + 2 * self.Hkv) * self.D
        from . import tp as tpmod
        shard_full = keep_reference and tp_size > 1      # parity runs: every rank builds the FULL weights, then slices
        for l in range(cfg.layers):
            base = (seed * 100003 + l) * 16 + (0 if shard_full else tp_rank * 7919)
            L = {}
            if shard_full:
                _, f0 = make_weight(H, (cfg.head_num + 2 * cfg.kv_head_num) * self.D, base + 1)
                _, f1 = make_weight(cfg.head_num * self.D, H, base + 2)
                _, f2 = make_weight(H, 2 * cfg.inter, base + 3)
                _, f3 = make_weight(cfg.inter, H, base + 4)
                r0 = tpmod.shard_qkv(f0, cfg.head_num, cfg.kv_head_num, self.D, tp_rank, tp_size)
                r1 = tpmod.shard_o(f1, cfg.head_num, self.D, tp_rank, tp_size)
                r2 = tpmod.shard_w13(f2, cfg.inter, tp_rank, tp_size)
                r3 = tpmod.shard_w2(f3, cfg.inter, tp_rank, tp_size)
                L["qkv"], L["o"], L["w2"] = pack_ref(r0), pack_ref(r1), pack_ref(r3)
                L["w13"] = pack_ref(r2, self.inter if self.fuse_silu else 0)
                L["full"] = dict(qkv=f0, o=f1, w13=f2, w2=f3)
            else:
                P = {}
                if act_order:
                    ga = torch.Generator().manual_seed(base + 9)
                    P = dict(qkv=torch.randperm(H, generator=ga), o=torch.randperm(self.Hq * self.D, generator=ga),
                             w13=torch.randperm(H, generator=ga), w2=torch.randperm(self.inter, generator=ga))
                    L["perm"] = P
                L["qkv"], r0 = make_weight(H, qkv_n, base + 1, perm=P.get("qkv"))
                L["o"], r1 = make_weight(self.Hq * self.D, H, base + 2, perm=P.get("o"))
                L["w13"], r2 = make_weight(H, 2 * self.inter, base + 3, gate_up_inter=self.inter if self.fuse_silu else 0,
                                           perm=P.get("w13"), col_perm=P.get("w2"))
                L["w2"], r3 = make_weight(self.inter, H, base + 4)
            L["ln1"] = (1.0 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(device)
            L["ln2"] = (1.0 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(device)
            L["kv"] = None
            if keep_reference:
                L["ref"] = dict(qkv=r0, o=r1, w13=r2, w2=r3)
            self.layers.append(L)
        self.final_ln = (1.0 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(device)
        if cfg.qk_norm:   # a generator of their own, so that no other weight moves; [D], replicated under TP
            gn = torch.Generator(device="cpu").manual_seed(seed * 1000 + 29)
            for L in self.layers:
                L["q_norm"] = (1.0 + 0.1 * torch.randn(self.D, generator=gn)).to(dtype).to(device)
                L["k_norm"] = (1.0 + 0.1 * torch.randn(self.D, generator=gn)).to(dtype).to(device)
        if shard_full:
            _, self.lm_head_full = make_weight(H, cfg.vocab, seed * 100003 + 999983, quant="f16")
            self.lm_head_ref = tpmod.shard_lm_head(self.lm_head_full, self.vocab, tp_rank)
            self.lm_head = pack_ref(self.lm_head_ref)
        else:
            self.lm_head, self.lm_head_ref = make_weight(H, self.vocab, seed * 100003 + 999983 + tp_rank, quant="f16")
        gg = torch.Generator(device=device).manual_seed(seed + 5)
        self.embed = (torch.randn(cfg.vocab, H, generator=gg, device=device) * 0.5).to(dtype)

        # ---- paged KV cache: P = B*M + 1 pages per layer, block 0 reserved, random permutation of the rest (SURVEY 8d)
        P = batch * self.M + 1
        gk = torch.Generator(device=device).manual_seed(42)
        for L in self.layers:
            if shard_full:
                # parity runs: the FULL pool (all kv heads) from a common seed, then this rank's heads -- every rank holds
                # DIFFERENT K/V, so a kv-head mix-up between ranks cannot cancel out against the unsharded oracle
                full = torch.randn(P, 2, cfg.kv_head_num, T, self.D, generator=gk, device=device).to(dtype)
                kv_rank = tp_rank if cfg.kv_head_num >= tp_size else tp_rank * cfg.kv_head_num // tp_size
                L["kv_full"] = full.cpu()
                L["kv"] = full[:, :, kv_rank * self.Hkv:(kv_rank + 1) * self.Hkv].contiguous()
            else:
                L["kv"] = torch.randn(P, 2, self.Hkv, T, self.D, generator=gk, device=device).to(dtype)
        gp = torch.Generator().manual_seed(3)
        perm = torch.randperm(P - 1, generator=gp).to(torch.int32) + 1
        self.block_ids_h = perm.reshape(batch, self.M).contiguous().pin_memory()
        if ragged:
            gl = torch.Generator().manual_seed(4)
            lens = torch.randint(ctx // 2, ctx + 1, (batch,), generator=gl)
        else:
            lens = torch.full((batch,), ctx)
        if beam_width > 1:    # one prompt per request, room for max_new_tokens
            lens = (lens.view(-1, beam_width)[:, :1].expand(-1, beam_width).reshape(-1) - max_new_tokens + 1).clamp(min=1)
        elif self.sample_advances:
            lens = (lens - max_new_tokens + 1).clamp(min=1)
        self.seq_lens_h = (lens - q_len).to(torch.int32).pin_memory()   # tokens already cached (SURVEY a3)
        self.ids_h = torch.randint(0, cfg.vocab, (batch,) if q_len == 1 else (batch, q_len), generator=gp).to(torch.int32).pin_memory()
        if beam_width > 1:
            self.own_pages = self.block_ids_h.clone()                 # every beam's private pages, by page-table index
            full = self.seq_lens_h.view(-1, beam_width)[:, 0] // T    # the prompt's full pages, shared by the request's beams
            blk = self.block_ids_h.view(-1, beam_width, self.M)
            for b in range(blk.shape[0]):
                f = int(full[b])
                blk[b, 1:, :f] = blk[b, 0, :f]
                if f < self.M:                                        # the prompt's partial page: the same tokens in every beam
                    for L in self.layers:
                        L["kv"][blk[b, 1:, f].long().to(device)] = L["kv"][int(blk[b, 0, f])].clone()
            self.ids_h.copy_(self.ids_h.view(-1, beam_width)[:, :1].expand(-1, beam_width).reshape(-1))
            self.shared_lens_h = (full * T).to(torch.int32).pin_memory()
        self.next_h = torch.zeros(batch, dtype=torch.int32).pin_memory()
        if q_len > 1:
            self.drafts_h = torch.zeros(batch, q_len - 1, dtype=torch.int32).pin_memory()
            self.out_tokens_h = torch.zeros(batch, q_len, dtype=torch.int32).pin_memory()
            self.accepted_h = torch.zeros(batch, dtype=torch.int32).pin_memory()

        # ---- static device buffers (graph-capturable: nothing is allocated inside step())
        def buf(*shape, dt=dtype):
            return torch.empty(*shape, dtype=dt, device=device)
        self.ids = buf(R, dt=torch.int32)
        self.seq_lens = buf(batch, dt=torch.int32)
        self.block_ids = buf(batch, self.M, dt=torch.int32)
        self.page_list = buf(batch, 1, 2, self.M, dt=torch.int32)
        self.resid = buf(R, H)
        self.x = buf(R, H)
        self.qkv = buf(R, qkv_n)
        self.q = buf(R, self.Hq * self.D)
        self.attn = buf(R, self.Hq * self.D)
        self.proj = buf(R, H)
        self.gu = buf(R, 2 * self.inter)
        self.act = buf(R, self.inter)
        self.logits = buf(R, self.vocab)
        self.logits_all = buf(tp_size, batch, self.vocab) if tp_size > 1 else None
        self.next_ids = buf(R, dt=torch.int32)                                # each row's greedy token
        if q_len > 1:
            self.drafts = buf(batch, q_len - 1, dt=torch.int32)
            self.out_tokens = buf(batch, q_len, dt=torch.int32)
            self.accepted = buf(batch, dt=torch.int32)
        if tree is not None:    # the token tree: parents and depths (pinned twins set_tree() fills), rotation positions, path
            self.tree_parents_h = torch.zeros(batch, q_len, dtype=torch.int32).pin_memory()
            self.tree_depth_h = torch.zeros(batch, q_len, dtype=torch.int32).pin_memory()
            self.tree_parents = buf(batch, q_len, dt=torch.int32)
            self.tree_depth = buf(batch, q_len, dt=torch.int32)
            self.tree_pos = buf(R, dt=torch.int32)
            self.accepted_path = buf(batch, q_len, dt=torch.int32)
            self.accepted_path_h = torch.zeros(batch, q_len, dtype=torch.int32).pin_memory()
        if beam_width > 1:
            W, B = beam_width, self.requests
            self.beam_cum = buf(B, W, dt=torch.float32)
            self.hist = buf(R, ctx, dt=torch.int32)
            self.hist_len = buf(R, dt=torch.int32)
            self.ngram_size = torch.full((R,), no_repeat_ngram, dtype=torch.int32, device=device)
            self.beam_out = {k: buf(B, n, dt=dt) for k, n, dt in (
                ("cand_token", 2 * W, torch.int32), ("cand_parent", 2 * W, torch.int32), ("cand_score", 2 * W, torch.float32),
                ("next_token", W, torch.int32), ("next_parent", W, torch.int32), ("next_cum", W, torch.float32))}
            self.beam_ws = ops.beam_search_workspace(B, W, self.vocab, device)
            self.own_pages_i32 = self.own_pages.to(device)
            self.own_pages_d = self.own_pages_i32.to(torch.int64)
            self.row_base = torch.arange(R, device=device) // W * W                  # row of beam 0 of each row's request
            self.row_m = torch.arange(R, device=device) * self.M
            self.page_idx = torch.arange(self.M, device=device)
            # fork scratch (static: the fork runs inside a CUDA graph)
            self.parent_row, self.pos = buf(R, dt=torch.int64), buf(R, dt=torch.int64)
            self.src_flat, self.dst_flat, self.pick_flat = (buf(R, dt=torch.int64) for _ in range(3))
            self.src_page, self.dst_page = buf(R, dt=torch.int64), buf(R, dt=torch.int64)
            self.partial = buf(R, dt=torch.bool)
            self.full_mask = buf(R, self.M, dt=torch.bool)
            self.blk_parent = buf(R, self.M, dt=torch.int32)
            self.hist_parent = buf(R, ctx, dt=torch.int32)
            self.len_parent = buf(R, dt=torch.int32)
            self.page_scratch = buf(R, 2, self.Hkv, T, self.D)
            self.shared_lens = buf(B, dt=torch.int32)
            if eos_id is not None:    # the finished-hypothesis sets (emptied by upload_inputs)
                self.hyp_state = ops.beam_hypotheses_state(B, W, max_new_tokens, device)
                self.done = torch.zeros(B, dtype=torch.int32, device=device)
                self.length_penalty = torch.tensor(alphas, dtype=torch.float32, device=device)
                self.early_stopping = torch.tensor(modes, dtype=torch.int32, device=device)
        if sampling is not None:
            def per_row(v, dt):
                t = torch.tensor(v if isinstance(v, (list, tuple)) else [v] * batch, dtype=dt)
                if t.numel() != batch:
                    raise ValueError(f"sampling: {len(v)} values for {batch} requests")
                return t.repeat_interleave(q_len).to(device)
            sp = sampling
            self.samp_params = dict(temperature=per_row(sp.temperature, torch.float32), top_k=per_row(sp.top_k, torch.int32),
                                    top_p=per_row(sp.top_p, torch.float32))
            if sp.has_penalties():
                self.samp_params.update(repetition=per_row(sp.repetition, torch.float32), presence=per_row(sp.presence, torch.float32),
                                        frequency=per_row(sp.frequency, torch.float32),
                                        count_ws=torch.zeros(R, self.vocab, dtype=torch.int32, device=device))
            if sp.has_min_p():
                self.samp_params["min_p"] = per_row(sp.min_p, torch.float32)
            self.samp_logits = buf(R, self.vocab, dt=torch.float32)
            self.token_prob = buf(R, dt=torch.float32)
            self.log_prob = buf(R, dt=torch.float32)
            self.uniform = buf(R if q_len == 1 else 2 * R, dt=torch.float32)
            self.draw_step = torch.zeros(1, dtype=torch.int64, device=device)
            self.uniforms = _Uniforms(sp.seed, self.uniform.numel(), device)
            if q_len == 1:
                self.cum_log_probs = buf(R, dt=torch.float32)
                self.hist = buf(R, ctx, dt=torch.int32)
                self.hist_len = buf(R, dt=torch.int32)
                self.ngram_size = torch.full((R,), no_repeat_ngram, dtype=torch.int32, device=device)
                self.hist_pos = buf(R, dt=torch.int64)
            else:
                self.target_probs = buf(batch, q_len, self.vocab, dt=torch.float32)
            if logprobs is not None:
                self.lp_out = dict(token_logprob=buf(R, dt=torch.float32), top_ids=buf(R, logprobs, dt=torch.int32),
                                   top_logprobs=buf(R, logprobs, dt=torch.float32))
                self.lp_ws = ops.token_logprobs_workspace(R, self.vocab, logprobs, device)
        # constrained decoding: device buffers the step reads, pinned host twins set_constraints() fills
        if token_bitmask:
            self.bitmask_h = torch.full((R, (self.vocab + 31) // 32), -1, dtype=torch.int32).pin_memory()
            self.bitmask = buf(R, self.bitmask_h.shape[1], dt=torch.int32)
        if logit_bias_capacity:
            self.bias_h = (torch.zeros(R + 1, dtype=torch.int32).pin_memory(),
                           torch.zeros(logit_bias_capacity, dtype=torch.int32).pin_memory(),
                           torch.zeros(logit_bias_capacity, dtype=torch.float32).pin_memory())
            self.bias = tuple(torch.zeros_like(t, device=device) for t in self.bias_h)
        self.x_perm = buf(R, H) if act_order else None                        # x[:, perm] before qkv / w13
        self.attn_perm = buf(R, self.Hq * self.D) if act_order else None      # attn[:, perm] before o
        shapes = [(H, qkv_n), (self.Hq * self.D, H), (H, 2 * self.inter), (self.inter, H), (H, self.vocab)]
        self.gemm_ws = ops.gemm_workspace(R, shapes, device)
        self.attn_ws = ops.attn_workspace(R, self.Hq, self.Hkv, ctx, device)
        rope.table(self.rope_spec, self.qkv.device)    # the cos/sin table is uploaded here, never inside a graph capture
        ops.set_pdl(pdl)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.prog = None
        if tree is not None:
            self.set_tree(tree)
        self.upload_inputs()
        torch.cuda.synchronize(device)

    # ------------------------------------------------------------------ host <-> device
    def upload_inputs(self):
        """H2D of one step's inputs from pinned host memory (token ids, lengths, block table)."""
        self.ids.copy_(self.ids_h.view(-1), non_blocking=True)
        self.seq_lens.copy_(self.seq_lens_h, non_blocking=True)
        self.block_ids.copy_(self.block_ids_h, non_blocking=True)
        if self.q_len > 1:
            self.drafts_h.copy_(self.ids_h[:, 1:])
            self.drafts.copy_(self.drafts_h, non_blocking=True)
        if self.W > 1:        # back to the prompt: beam 0 alone live (cum 0), the input token as the whole history
            self.shared_lens.copy_(self.shared_lens_h, non_blocking=True)
            self.beam_cum.fill_(-math.inf)
            self.beam_cum[:, 0] = 0.0
            self.hist[:, 0].copy_(self.ids)
            self.hist_len.fill_(1)
            self.beam_steps = 0
            if self.eos_id is not None:
                self.hyp_state.zero_()
                self.done.zero_()
        if self.samp is not None:  # back to the prompt: step 0 of the uniforms; at q_len 1 the input token as the whole history
            self.draw_step.zero_()
            if self.q_len == 1:
                self.cum_log_probs.zero_()
                self.hist[:, 0].copy_(self.ids)
                self.hist_len.fill_(1)
                self.beam_steps = 0
        if self.bitmask is not None or self.bias is not None:
            self.set_constraints()

    def set_constraints(self, bitmask=None, logit_bias: Optional[Sequence[Mapping[int, float]]] = None):
        """The constraints the next step (or graph replay) applies, from host data, copied non_blocking into the static
        buffers: bitmask int32 [R, ceil(V / 32)] (numpy or CPU tensor, xgrammar's layout; None: every token allowed) and
        logit_bias, one {token id: bias} mapping per logits row (None: no bias; at most logit_bias_capacity entries in all).
        R is the step's logits rows: row b (greedy, sampling), b * q_len + j (verification: position j), b * W + i (beam i).
        Like upload_inputs(), it rewrites pinned buffers a copy may still read: call it once the previous step has been
        enqueued and its inputs are no longer needed, as between two replays."""
        R, V = self.B * self.q_len, self.vocab
        if bitmask is not None:
            if self.bitmask is None:
                raise ValueError("set_constraints: this step was built without token_bitmask=True")
            m = torch.as_tensor(bitmask)
            if m.dtype != torch.int32 or tuple(m.shape) != tuple(self.bitmask_h.shape) or m.device.type != "cpu":
                raise ValueError(f"set_constraints: bitmask must be host int32 {list(self.bitmask_h.shape)} (got {m.dtype} "
                                 f"{list(m.shape)} on {m.device})")
        if logit_bias is not None:
            if self.bias is None:
                raise ValueError("set_constraints: this step was built without logit_bias_capacity")
            if len(logit_bias) != R:
                raise ValueError(f"set_constraints: logit_bias needs one mapping per logits row ({R}, got {len(logit_bias)})")
            try:
                offsets, ids, values = ops.logit_bias_csr(logit_bias, V)
            except ops.B200Error as e:
                raise ValueError(str(e)) from None
            if ids.numel() > self.bias_h[1].numel():
                raise ValueError(f"set_constraints: {ids.numel()} logit_bias entries exceed logit_bias_capacity "
                                 f"{self.bias_h[1].numel()}")
        if self.bitmask is not None:
            if bitmask is None:
                self.bitmask_h.fill_(-1)
            else:
                self.bitmask_h.copy_(m)
            self.bitmask.copy_(self.bitmask_h, non_blocking=True)
        if self.bias is not None:
            if logit_bias is None:
                self.bias_h[0].zero_()
            else:
                self.bias_h[0].copy_(offsets)
                self.bias_h[1][:ids.numel()] = ids
                self.bias_h[2][:ids.numel()] = values
            for d, h in zip(self.bias, self.bias_h):
                d.copy_(h, non_blocking=True)

    def set_tree(self, parents):
        """The token tree the next step (or graph replay) verifies: one parent list for every request, or one per request, of
        q_len entries (parents[0] = -1 for the root, 0 <= parents[j] < j). Fills the pinned twins of the static parent and depth
        buffers and copies them non_blocking, like set_constraints(): call it between two replays."""
        if self.tree_parents is None:
            raise ValueError("set_tree: this step was built without tree=")
        n, B = self.q_len, self.B
        rows = [list(parents)] * B if len(parents) == 0 or not isinstance(parents[0], (list, tuple)) else [list(r) for r in parents]
        if len(rows) != B:
            raise ValueError(f"set_tree: {len(rows)} parent lists for {B} requests")
        depth = []
        for r in rows:
            if len(r) != n or int(r[0]) != -1 or any(not 0 <= int(r[j]) < j for j in range(1, n)):
                raise ValueError(f"set_tree: parents must hold {n} entries, -1 for the root and 0 <= parents[j] < j (got {r})")
            d = [0] * n
            for j in range(1, n):
                d[j] = d[int(r[j])] + 1
            depth.append(d)
        self.tree_parents_h.copy_(torch.tensor(rows, dtype=torch.int32))
        self.tree_depth_h.copy_(torch.tensor(depth, dtype=torch.int32))
        self.tree_parents.copy_(self.tree_parents_h, non_blocking=True)
        self.tree_depth.copy_(self.tree_depth_h, non_blocking=True)

    def _constrain(self, logits: torch.Tensor):
        """b200_constrain_logits on `logits` with the buffers set_constraints() filled (no launch when the step has none)."""
        if self.bitmask is not None or self.bias is not None:
            ops.constrain_logits(logits, bitmask=self.bitmask, logit_bias=self.bias)

    sample_advances = False
    bitmask = bitmask_h = bias = bias_h = None     # no constraint buffers unless token_bitmask / logit_bias_capacity
    tree_parents = None                             # no token tree unless tree=

    def _count_beam_step(self):
        if self.W > 1 or self.sample_advances:
            if self.beam_steps >= self.max_new_tokens:
                raise ValueError(f"step {self.beam_steps + 1} since the prompt exceeds max_new_tokens {self.max_new_tokens}: "
                                 "call upload_inputs() to restart from the prompt")
            self.beam_steps += 1

    def download_outputs(self):
        if self.q_len > 1:
            self.out_tokens_h.copy_(self.out_tokens, non_blocking=True)
            self.accepted_h.copy_(self.accepted, non_blocking=True)
            if self.tree_parents is not None:
                self.accepted_path_h.copy_(self.accepted_path, non_blocking=True)
            return
        self.next_h.copy_(self.beam_out["next_token"].view(-1) if self.W > 1 else self.next_ids, non_blocking=True)

    def h2d_bytes(self) -> int:
        drafts = self.drafts_h.numel() * 4 if self.q_len > 1 else 0
        constraints = sum(t.numel() * 4 for t in ([self.bitmask_h] if self.bitmask is not None else [])
                          + (list(self.bias_h) if self.bias is not None else []))
        return self.ids_h.numel() * 4 + self.seq_lens_h.numel() * 4 + self.block_ids_h.numel() * 4 + drafts + constraints

    def d2h_bytes(self) -> int:
        if self.q_len > 1:
            return self.out_tokens_h.numel() * 4 + self.accepted_h.numel() * 4
        return self.next_h.numel() * 4

    # ------------------------------------------------------------------ the step
    def _all_reduce(self, t: torch.Tensor):
        if self.tp_size > 1:
            self.comm.all_reduce(t)

    def _row_gemm(self, x, w):
        """self.proj = x . w for a row-parallel weight (o, w2). Fused form (b200_wo_gemm_rs): the GEMM epilogue pushes the
        reduce-scatter words over NVLink; the _ar_norm() that follows then only reduces / gathers / normalises."""
        if self.fuse_gemm_rs and hasattr(self.comm, "gemm_rs"):    # (bench.py swaps the communicator for its NCCL parity arm)
            self.comm.gemm_rs(x, w, self.gemm_ws, self.proj, pdl=self.pdl)
        else:
            ops.wo_gemm(x, w, self.gemm_ws, out=self.proj, pdl=self.pdl, x_perm=self.attn_perm)

    def _ar_norm(self, t, gamma):
        """[TP all-reduce of the row-parallel GEMM output t] + residual add + RMSNorm -> self.x. With the peer communicator the
        three steps are ONE kernel (b200_peer_allreduce_norm); otherwise all-reduce and fused_add_rmsnorm run separately."""
        if self.fuse_gemm_rs and hasattr(self.comm, "gemm_rs"):      # t came out of _row_gemm(): its scatter phase is already on the wire
            self.comm.gather_norm(t, self.resid, gamma, self.cfg.eps, self.x)
            return
        if self.tp_size > 1:
            fused = getattr(self.comm, "all_reduce_norm", None)
            if self.fuse_ar_norm and fused is not None and fused(t, self.resid, gamma, self.cfg.eps, self.x):
                return
            self.comm.all_reduce(t)
        ops.add_rmsnorm(t, self.resid, gamma, self.cfg.eps, out=self.x)

    def _rope_append(self, L):
        """q of the step's rows into self.q, their K/V into layer L's cache: rope.rope_append, with L's QK-norm when the config
        has one."""
        qk_norm = (L["q_norm"], L["k_norm"], self.cfg.eps) if self.cfg.qk_norm else None
        pos = self.tree_pos if self.tree_parents is not None else None   # (tree mode: seq + depth, formed in step_core)
        rope.rope_append(self.rope_spec, self.qkv, L["kv"], self.page_list, self.seq_lens, self.Hq, q_out=self.q, q_len=self.q_len,
                         qk_norm=qk_norm, position_ids=pos)

    def _attention(self, L):
        """self.attn = the attention of the step's rows over layer L's cache, after _rope_append. In beam mode a request's beams
        share one pass over its prompt when their rows fit (attention.beam_rows_fit)."""
        if self.tree_parents is not None:    # each node attends to the cache and its ancestors
            ops.paged_decode_attn_tree(self.q.view(self.B, self.q_len, self.Hq, self.D), L["kv"], self.page_list, self.seq_lens,
                                       self.tree_parents, self.ctx, self.attn_ws, out=self.attn.view(self.B, self.q_len, self.Hq * self.D))
        elif self.q_len > 1:    # each query token attends up to its own position
            ops.paged_decode_attn_multi(self.q.view(self.B, self.q_len, self.Hq, self.D), L["kv"], self.page_list, self.seq_lens,
                                        self.ctx, self.attn_ws, out=self.attn.view(self.B, self.q_len, self.Hq * self.D))
        elif beam_rows_fit(self.Hq, self.Hkv, self.W, self.requests):
            ops.paged_decode_attn_beam(self.q.view(self.requests, self.W, self.Hq, self.D), L["kv"], self.page_list, self.seq_lens,
                                       self.shared_lens, self.ctx, self.attn_ws,
                                       out=self.attn.view(self.requests, self.W, self.Hq * self.D))
        else:
            ops.paged_decode_attn(self.q, L["kv"], self.page_list, self.seq_lens, self.ctx, self.attn_ws, out=self.attn)

    def step_core(self):
        """Everything up to the sampled token (TP1 / peer communicator) or the local logits (NCCL): C-ABI calls only, so it
        can be recorded into a decode program."""
        cfg = self.cfg
        ops.convert_block_table(self.block_ids, out=self.page_list)
        if self.tree_parents is not None:    # node j is rotated at seq + depth(j) (its K/V still go to slot seq + j)
            torch.add(self.seq_lens.view(-1, 1), self.tree_depth, out=self.tree_pos.view(self.B, self.q_len))
        ops.embedding(self.ids, self.embed, out=self.resid)
        first = True
        for L in self.layers:
            if first:
                ops.add_rmsnorm(self.resid, None, L["ln1"], cfg.eps, out=self.x)
                first = False
            else:
                self._ar_norm(self.proj, L["ln1"])          # all-reduce of the previous layer's w2 output rides along
            ops.wo_gemm(self.x, L["qkv"], self.gemm_ws, out=self.qkv, pdl=self.pdl, x_perm=self.x_perm)
            if self.fuse_rope:    # RoPE + K/V append inside the attention kernel (one launch instead of two)
                ops.paged_decode_attn_rope(self.qkv, L["kv"], self.page_list, self.seq_lens, self.Hq, self.ctx,
                                           self.rope_spec.base, self.attn_ws, out=self.attn)
            else:                 # K/V of the step's tokens appended, then the attention over the cache
                self._rope_append(L)
                self._attention(L)
            self._row_gemm(self.attn, L["o"])
            self._ar_norm(self.proj, L["ln2"])
            if self.fuse_silu:     # SiLU(gate)*up in the GEMM epilogue (gate/up columns interleaved at load time)
                ops.wo_gemm(self.x, L["w13"], self.gemm_ws, out=self.act, pdl=self.pdl, silu_mul=True, x_perm=self.x_perm)
            else:
                ops.wo_gemm(self.x, L["w13"], self.gemm_ws, out=self.gu, pdl=self.pdl, x_perm=self.x_perm)
                ops.silu_and_mul(self.gu, out=self.act)
            self._row_gemm(self.act, L["w2"])
        self._ar_norm(self.proj, self.final_ln)
        ops.wo_gemm(self.x, self.lm_head, self.gemm_ws, out=self.logits, pdl=self.pdl)
        if self.W > 1:
            self._constrain(self.logits)
            if self.ngram > 0:
                ops.ban_repeat_ngram(self.logits, self.hist, self.hist_len, self.ngram_size)
            ops.beam_search_step(self.logits, self.beam_cum, self.W, eos_id=-1 if self.eos_id is None else self.eos_id,
                                 workspace=self.beam_ws, out=self.beam_out)
            if self.eos_id is not None:    # between the beam step and the fork: the history rows are still the parents'
                ops.beam_hypotheses_update(self.beam_out, self.hist, self.hist_len, self.eos_id, self.length_penalty,
                                           self.early_stopping, self.hyp_state, self.done, self.max_new_tokens, gen_start=1)
            self.fork()
        elif self.samp is not None:
            self.sample()
        elif self.tp_size == 1:
            self._constrain(self.logits)
            ops.argmax(self.logits, out=self.next_ids)
            if self.tree_parents is not None:
                self._verify_tree(target_ids=self.next_ids.view(self.B, self.q_len))
            elif self.q_len > 1:
                ops.spec_verify(self.drafts, target_ids=self.next_ids.view(self.B, self.q_len), out_tokens=self.out_tokens,
                                accepted=self.accepted)
        elif hasattr(self.comm, "argmax"):
            self.comm.argmax(self.logits, cfg.vocab, self.next_ids)     # vocab-parallel greedy sampling, own kernel

    def fork(self):
        """Beam mode, after beam_search_step: every row becomes the new beam of its slot (see the class docstring). Torch index
        ops on static buffers only, so a CUDA graph replays it."""
        o, T, M, cap = self.beam_out, self.cfg.tokens_per_block, self.M, self.hist.shape[1]
        torch.add(self.row_base, o["next_parent"].view(-1), out=self.parent_row)
        self.beam_cum.copy_(o["next_cum"])
        # token history: the parent's row, then the new token
        torch.index_select(self.hist, 0, self.parent_row, out=self.hist_parent)
        torch.index_select(self.hist_len, 0, self.parent_row, out=self.len_parent)
        self.hist.copy_(self.hist_parent)
        self.pos.copy_(self.len_parent)
        self.pos.clamp_(max=cap - 1)
        self.hist.scatter_(1, self.pos.view(-1, 1), o["next_token"].view(-1, 1))
        self.hist_len.copy_(self.pos)
        self.hist_len.add_(1)
        # page table: the parent's entries for the pages the step filled (q = (seq + 1) // T of them), the own pages after them
        self.pos.copy_(self.seq_lens)
        self.pos.add_(1)
        self.pos.floor_divide_(T)
        torch.lt(self.page_idx.view(1, -1), self.pos.view(-1, 1), out=self.full_mask)
        torch.index_select(self.block_ids, 0, self.parent_row, out=self.blk_parent)
        torch.where(self.full_mask, self.blk_parent, self.own_pages_i32, out=self.block_ids)
        # the parent's partial page q into the own page q, two-phase (a parent may be another row's child); with no partial
        # page (q == M) every row copies its own page onto itself
        torch.lt(self.pos, M, out=self.partial)
        self.pos.clamp_(max=M - 1)
        torch.add(self.row_m, self.pos, out=self.dst_flat)
        torch.mul(self.parent_row, M, out=self.src_flat)
        self.src_flat.add_(self.pos)
        torch.where(self.partial, self.src_flat, self.dst_flat, out=self.pick_flat)
        own = self.own_pages_d.view(-1)
        torch.index_select(own, 0, self.pick_flat, out=self.src_page)
        torch.index_select(own, 0, self.dst_flat, out=self.dst_page)
        for L in self.layers:
            torch.index_select(L["kv"], 0, self.src_page, out=self.page_scratch)
            L["kv"].index_copy_(0, self.dst_page, self.page_scratch)
        self.ids.copy_(o["next_token"].view(-1))
        self.seq_lens.add_(1)

    def beam_results(self, n: int) -> Dict[str, torch.Tensor]:
        """Beam mode with eos_id: the n (1..W) best hypotheses of each request now (beam_hypotheses_finalize on the current state,
        which it leaves as it is), as host tensors: tokens int32 [B, n, max_new_tokens] (the generated tokens, -1 past each
        path), len int32 [B, n], score / cum fp32 [B, n]."""
        if self.W == 1 or self.eos_id is None:
            raise ValueError("beam_results needs the beam mode with an eos_id")
        out = ops.beam_hypotheses_finalize(self.hyp_state, self.done, self.beam_cum, self.hist, self.hist_len, n, self.max_new_tokens,
                                           self.length_penalty, gen_start=1)
        return {k: v.cpu() for k, v in out.items()}

    def sample(self):
        """Sampling mode, after the lm_head (see the class docstring). b200 kernels and torch ops on static buffers only, so a CUDA
        graph replays it."""
        R, sp = self.B * self.q_len, self.samp_params
        self.uniforms.draw(self.draw_step, self.uniform)
        self.draw_step.add_(1)
        self.samp_logits.copy_(self.logits)
        self._constrain(self.samp_logits)
        adv = self.q_len == 1
        if adv and self.ngram > 0:
            ops.ban_repeat_ngram(self.samp_logits, self.hist, self.hist_len, self.ngram_size)
        hist = dict(history=self.hist, hist_len=self.hist_len) if adv else {}
        ops.sample(self.samp_logits, sp["top_k"], sp["top_p"], self.uniform[:R], temperature=sp["temperature"],
                   repetition=sp.get("repetition"), presence=sp.get("presence"), frequency=sp.get("frequency"),
                   count_ws=sp.get("count_ws"), min_p=sp.get("min_p"), out=dict(token=self.next_ids, token_prob=self.token_prob,
                                                         **({} if adv else dict(probs=self.target_probs))), **hist)
        if self.logprobs is not None:
            ops.token_logprobs(self.logits, self.logprobs, tokens=self.next_ids, workspace=self.lp_ws, out=self.lp_out)
        if not adv:
            if self.tree_parents is not None:
                self._verify_tree(target_probs=self.target_probs, uniform=self.uniform[R:])
            else:
                ops.spec_verify(self.drafts, target_probs=self.target_probs, uniform=self.uniform[R:], out_tokens=self.out_tokens,
                                accepted=self.accepted)
            return
        torch.log(self.token_prob, out=self.log_prob)
        self.cum_log_probs.add_(self.log_prob)
        self.hist_pos.copy_(self.hist_len)
        self.hist_pos.clamp_(max=self.hist.shape[1] - 1)
        self.hist.scatter_(1, self.hist_pos.view(-1, 1), self.next_ids.view(-1, 1))
        self.hist_len.add_(1)
        self.ids.copy_(self.next_ids)
        self.seq_lens.add_(1)

    def _verify_tree(self, **target):
        """Tree mode's ending: spec_verify_tree over the node tokens (the step's input ids; the root's is not read), then the
        accepted path's K/V moved to slots seq .. seq + accepted in every layer (one kv_compact_path launch)."""
        ops.spec_verify_tree(self.tree_parents, self.ids.view(self.B, self.q_len), out_tokens=self.out_tokens, accepted=self.accepted,
                             accepted_path=self.accepted_path, **target)
        ops.kv_compact_path([L["kv"] for L in self.layers], self.page_list, self.seq_lens, self.accepted_path, self.accepted)

    def step_tail(self):
        """TP > 1 with stock NCCL: gather the vocab-split logits and sample (torch plumbing, outside the program)."""
        if self.tp_size > 1 and not hasattr(self.comm, "argmax"):
            self.comm.all_gather(self.logits_all, self.logits)
            full = self.logits_all.permute(1, 0, 2).reshape(self.B, -1)[:, : self.cfg.vocab]   # drop the sp_0_pad8 columns
            self.next_ids.copy_(torch.argmax(full.float(), dim=-1).to(torch.int32))

    def step(self):
        """One decode step, op by op (one kernel per call)."""
        self._count_beam_step()
        self.step_core()
        self.step_tail()

    def build_program(self):
        """Record step_core() into a decode program (b200_program_*): the ops between two attention calls become one
        persistent-kernel launch. Requires every call in step_core to go through the C ABI (own peer all-reduce, not NCCL)."""
        from . import tp as tpmod
        assert self.tp_size == 1 or isinstance(self.comm, tpmod.PeerComm), "a program cannot record NCCL calls"
        if self.q_len > 1:
            raise ValueError("a verification step (q_len > 1) runs op by op or under a CUDA graph, not as a decode program")
        if self.W > 1:
            raise ValueError("a beam-search step runs op by op or under a CUDA graph, not as a decode program (its fork is "
                             "torch index ops, not C-ABI calls)")
        if self.samp is not None:
            raise ValueError("a sampling step runs op by op or under a CUDA graph, not as a decode program (its uniforms and "
                             "state updates are torch ops, not C-ABI calls)")
        self.prog = ops.Program()
        with self.prog.record():
            self.step_core()
        return self.prog

    def run(self):
        """One decode step through the program if one was built, else op by op."""
        if getattr(self, "prog", None) is not None:
            self.prog.launch()
            self.step_tail()
        else:
            self.step()

    def launches_per_step(self) -> int:
        n0 = ops.launch_count()
        self.run()
        return ops.launch_count() - n0

    def capture(self):
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            for _ in range(2):
                self.run()
                if self.W > 1 or self.samp is not None:   # the state / the draw counter advance: every warm-up starts from the prompt
                    self.upload_inputs()
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.run()
        if self.W > 1 or self.samp is not None:
            self.upload_inputs()            # the recorded step has not run: the first replay is step 1
        torch.cuda.synchronize(self.dev)

    def replay(self):
        self._count_beam_step()
        self.graph.replay()

    # ------------------------------------------------------------------ accounting (SURVEY 8d)
    def algorithmic_bytes(self) -> Dict[str, float]:
        cfg, H = self.cfg, self.cfg.hidden
        qkv_n = (self.Hq + 2 * self.Hkv) * self.D
        w = (weight_bytes(cfg, H, qkv_n) + weight_bytes(cfg, self.Hq * self.D, H) + weight_bytes(cfg, H, 2 * self.inter)
             + weight_bytes(cfg, self.inter, H)) * cfg.layers
        lens = (self.seq_lens_h.to(torch.int64) + self.q_len).sum().item()
        if self.W > 1:    # a request's shared prompt pages are one copy of K/V, whichever kernel reads them
            lens -= (self.W - 1) * self.shared_lens_h.to(torch.int64).sum().item()
        kv = 2.0 * lens * self.Hkv * self.D * 2 * cfg.layers
        lm = 2.0 * H * self.vocab
        return dict(weights=w, kv=kv, lm_head=lm, total=w + kv + lm)
