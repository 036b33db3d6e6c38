"""DecodeStep's option checks, without a GPU: every option set in CASES gets the outcome written beside it. A rejected set
raises ValueError before anything is allocated; its message is compared word for word, so for a set with several faults
the table also pins which check comes first. An accepted set gets as far as packing the first weight, which needs CUDA
tensors (B200Error)."""
import dataclasses

import pytest
import torch

from rtp_llm_b200._lib import B200Error
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams

ACCEPTED = "accepted"
F16 = dataclasses.replace(TINY, quant="f16")
SP = SamplingParams(temperature=0.8, top_k=5, top_p=0.9)
PEN = SamplingParams(repetition=1.2, presence=[0.0, 0.5, 0.0, 0.0])
MINP = SamplingParams(min_p=0.05)
BAD_MINP = SamplingParams(min_p=[0.0, 0.2, 1.1, 0.0])
TREE = [-1, 0, 0]

# (batch, options, outcome) of DecodeStep(options.get("cfg", TINY), batch, 40, cpu, **options)
CASES = [
    (4, dict(), ACCEPTED),
    (256, dict(), ACCEPTED),
    (257, dict(),
     'a step runs at most 256 token rows (the GEMM row limit), and at most 128 with tp_size > 1 (got 257 rows, tp_size'
     ' 1)'),
    (128, dict(tp_size=2), ACCEPTED),
    (129, dict(tp_size=2),
     'a step runs at most 256 token rows (the GEMM row limit), and at most 128 with tp_size > 1 (got 129 rows, tp_size'
     ' 2)'),
    (4, dict(max_rows=0), 'max_rows must be in 1..256, the GEMM row limit (got 0)'),
    (4, dict(max_rows=257), 'max_rows must be in 1..256, the GEMM row limit (got 257)'),
    (257, dict(max_rows=0), 'max_rows must be in 1..256, the GEMM row limit (got 0)'),
    (4, dict(q_len=0), 'q_len must be >= 1 (got 0)'),
    (4, dict(q_len=0, max_rows=0), 'max_rows must be in 1..256, the GEMM row limit (got 0)'),
    (4, dict(q_len=0, tree=TREE), 'q_len must be >= 1 (got 0)'),
    (4, dict(q_len=2), ACCEPTED),
    (64, dict(q_len=2), ACCEPTED),
    (65, dict(q_len=2),
     'a verification step (q_len 2) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 65, tp_size 1)'),
    (65, dict(q_len=2, max_rows=256), ACCEPTED),
    (129, dict(q_len=2, max_rows=256),
     'a verification step (q_len 2) needs batch * q_len <= 256 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 129, tp_size 1)'),
    (4, dict(q_len=2, tp_size=2),
     'a verification step (q_len 2) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 4, tp_size 2)'),
    (4, dict(q_len=2, max_rows=300), 'max_rows must be in 1..256, the GEMM row limit (got 300)'),
    (65, dict(q_len=2, beam_width=33),
     'a verification step (q_len 2) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 65, tp_size 1)'),
    (4, dict(q_len=2, beam_width=2),
     'beam search (beam_width 2) needs batch * beam_width <= 128 (max_rows; the GEMM row limit is 256), tp_size 1 and '
     'q_len 1 (got batch 4, tp_size 1, q_len 2)'),
    (40, dict(q_len=2, beam_width=2),
     'beam search (beam_width 2) needs batch * beam_width <= 128 (max_rows; the GEMM row limit is 256), tp_size 1 and '
     'q_len 1 (got batch 40, tp_size 1, q_len 2)'),
    (65, dict(q_len=2, beam_width=2),
     'a verification step (q_len 2) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 65, tp_size 1)'),
    (4, dict(q_len=2, beam_width=2, tp_size=2),
     'a verification step (q_len 2) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 4, tp_size 2)'),
    (4, dict(q_len=3, tree=TREE), ACCEPTED),
    (80, dict(q_len=3, tree=TREE, max_rows=256), ACCEPTED),
    (86, dict(q_len=3, tree=TREE, max_rows=256),
     'a verification step (q_len 3) needs batch * q_len <= 256 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 86, tp_size 1)'),
    (4, dict(q_len=1, tree=[-1]), 'a token-tree step needs q_len >= 2 nodes (got q_len 1)'),
    (4, dict(q_len=1, tree=[-1], beam_width=33), 'a token-tree step needs q_len >= 2 nodes (got q_len 1)'),
    (4, dict(q_len=3, tree=TREE, sampling=SP), ACCEPTED),
    (4, dict(q_len=3, tree=TREE, sampling=PEN),
     "sampled verification (q_len > 1) takes no penalties and no n-gram ban: row j's history would have to hold drafts"
     ' 0..j-1'),
    (4, dict(beam_width=2), ACCEPTED),
    (4, dict(beam_width=0), 'beam_width must be in 1..32 (got 0)'),
    (4, dict(beam_width=33), 'beam_width must be in 1..32 (got 33)'),
    (4, dict(beam_width=33, tp_size=2), 'beam_width must be in 1..32 (got 33)'),
    (32, dict(beam_width=4), ACCEPTED),
    (33, dict(beam_width=4),
     'beam search (beam_width 4) needs batch * beam_width <= 128 (max_rows; the GEMM row limit is 256), tp_size 1 and '
     'q_len 1 (got batch 33, tp_size 1, q_len 1)'),
    (64, dict(beam_width=4, max_rows=256), ACCEPTED),
    (65, dict(beam_width=4, max_rows=256),
     'beam search (beam_width 4) needs batch * beam_width <= 256 (max_rows; the GEMM row limit is 256), tp_size 1 and '
     'q_len 1 (got batch 65, tp_size 1, q_len 1)'),
    (4, dict(beam_width=2, tp_size=2),
     'beam search (beam_width 2) needs batch * beam_width <= 128 (max_rows; the GEMM row limit is 256), tp_size 1 and '
     'q_len 1 (got batch 4, tp_size 2, q_len 1)'),
    (4, dict(beam_width=2, no_repeat_ngram=3), ACCEPTED),
    (4, dict(beam_width=2, max_new_tokens=40), 'max_new_tokens must be in 1..ctx-1 (got 40, ctx 40)'),
    (4, dict(beam_width=2, max_new_tokens=0), 'max_new_tokens must be in 1..ctx-1 (got 0, ctx 40)'),
    (4, dict(beam_width=2, max_new_tokens=39), ACCEPTED),
    (4, dict(sampling=SP), ACCEPTED),
    (4, dict(sampling=SP, tp_size=2),
     'sampling needs tp_size 1, beam_width 1 and batch * q_len <= 128 (max_rows; the GEMM row limit is 256) (got '
     'tp_size 2, beam_width 1, batch 4, q_len 1)'),
    (129, dict(sampling=SP, tp_size=2),
     'sampling needs tp_size 1, beam_width 1 and batch * q_len <= 128 (max_rows; the GEMM row limit is 256) (got '
     'tp_size 2, beam_width 1, batch 129, q_len 1)'),
    (4, dict(sampling=SP, beam_width=2),
     'sampling needs tp_size 1, beam_width 1 and batch * q_len <= 128 (max_rows; the GEMM row limit is 256) (got '
     'tp_size 1, beam_width 2, batch 4, q_len 1)'),
    (4, dict(sampling=SP, beam_width=2, tp_size=2),
     'beam search (beam_width 2) needs batch * beam_width <= 128 (max_rows; the GEMM row limit is 256), tp_size 1 and '
     'q_len 1 (got batch 4, tp_size 2, q_len 1)'),
    (129, dict(sampling=SP),
     'sampling needs tp_size 1, beam_width 1 and batch * q_len <= 128 (max_rows; the GEMM row limit is 256) (got '
     'tp_size 1, beam_width 1, batch 129, q_len 1)'),
    (200, dict(sampling=SP, max_rows=256), ACCEPTED),
    (257, dict(sampling=SP, max_rows=256),
     'sampling needs tp_size 1, beam_width 1 and batch * q_len <= 256 (max_rows; the GEMM row limit is 256) (got '
     'tp_size 1, beam_width 1, batch 257, q_len 1)'),
    (33, dict(sampling=SP, q_len=4),
     'a verification step (q_len 4) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 33, tp_size 1)'),
    (4, dict(sampling=SP, q_len=2), ACCEPTED),
    (4, dict(sampling=SP, q_len=2, tp_size=2),
     'a verification step (q_len 2) needs batch * q_len <= 128 (max_rows; the GEMM row limit is 256) and tp_size 1 '
     '(got batch 4, tp_size 2)'),
    (4, dict(sampling=PEN, q_len=2),
     "sampled verification (q_len > 1) takes no penalties and no n-gram ban: row j's history would have to hold drafts"
     ' 0..j-1'),
    (4, dict(sampling=SP, q_len=2, no_repeat_ngram=2),
     "sampled verification (q_len > 1) takes no penalties and no n-gram ban: row j's history would have to hold drafts"
     ' 0..j-1'),
    (4, dict(sampling=PEN, q_len=2, logprobs=65),
     "sampled verification (q_len > 1) takes no penalties and no n-gram ban: row j's history would have to hold drafts"
     ' 0..j-1'),
    (4, dict(sampling=PEN, q_len=2, max_new_tokens=40),
     "sampled verification (q_len > 1) takes no penalties and no n-gram ban: row j's history would have to hold drafts"
     ' 0..j-1'),
    (4, dict(sampling=PEN, logprobs=5, no_repeat_ngram=2), ACCEPTED),
    (4, dict(sampling=SP, logprobs=0), ACCEPTED),
    (4, dict(sampling=SP, logprobs=64), ACCEPTED),
    (4, dict(sampling=SP, logprobs=65), 'logprobs must be in 0..64 (got 65)'),
    (4, dict(sampling=SP, logprobs=-1), 'logprobs must be in 0..64 (got -1)'),
    (4, dict(sampling=SP, logprobs=65, max_new_tokens=40), 'logprobs must be in 0..64 (got 65)'),
    (4, dict(sampling=SP, max_new_tokens=40), 'max_new_tokens must be in 1..ctx-1 (got 40, ctx 40)'),
    (4, dict(sampling=SP, q_len=2, max_new_tokens=40), ACCEPTED),
    (4, dict(sampling=MINP), ACCEPTED),
    (4, dict(sampling=BAD_MINP), 'sampling: min_p must be in [0, 1] (got [0.0, 0.2, 1.1, 0.0])'),
    (4, dict(sampling=SamplingParams(min_p=1.5), max_rows=0), 'sampling: min_p must be in [0, 1] (got 1.5)'),
    (4, dict(sampling=SamplingParams(min_p=-0.1), token_bitmask=True, tp_size=2),
     'token_bitmask / logit_bias need tp_size 1 (got tp_size 2): the vocabulary-parallel argmax would need a mask '
     'sharded by vocabulary'),
    (4, dict(logprobs=5), 'logprobs needs the sampling mode (sampling=SamplingParams(...))'),
    (4, dict(logprobs=5, beam_width=2, max_new_tokens=40), 'logprobs needs the sampling mode (sampling=SamplingParams(...))'),
    (4, dict(logprobs=5, no_repeat_ngram=3), 'logprobs needs the sampling mode (sampling=SamplingParams(...))'),
    (257, dict(logprobs=5), 'logprobs needs the sampling mode (sampling=SamplingParams(...))'),
    (4, dict(max_new_tokens=40), ACCEPTED),
    (4, dict(no_repeat_ngram=3), 'no_repeat_ngram 3 needs beam search (beam_width > 1); the greedy step has no ban'),
    (4, dict(no_repeat_ngram=3, eos_id=5), 'no_repeat_ngram 3 needs beam search (beam_width > 1); the greedy step has no ban'),
    (257, dict(no_repeat_ngram=3), 'no_repeat_ngram 3 needs beam search (beam_width > 1); the greedy step has no ban'),
    (4, dict(eos_id=5), 'eos_id needs beam search (beam_width > 1) and must be in 0..vocab-1 (got eos_id 5, beam_width 1)'),
    (4, dict(eos_id=5, length_penalty=[1.0, 1.0, 1.0]),
     'eos_id needs beam search (beam_width > 1) and must be in 0..vocab-1 (got eos_id 5, beam_width 1)'),
    (4, dict(beam_width=2, eos_id=5), ACCEPTED),
    (4, dict(beam_width=2, eos_id=TINY.vocab),
     'eos_id needs beam search (beam_width > 1) and must be in 0..vocab-1 (got eos_id 1024, beam_width 2)'),
    (4, dict(beam_width=2, eos_id=-1),
     'eos_id needs beam search (beam_width > 1) and must be in 0..vocab-1 (got eos_id -1, beam_width 2)'),
    (4, dict(beam_width=2, eos_id=TINY.vocab, max_new_tokens=40), 'max_new_tokens must be in 1..ctx-1 (got 40, ctx 40)'),
    (4, dict(beam_width=2, eos_id=5, length_penalty=[1.0, 1.0, 1.0]), 'length_penalty: 3 values for 4 requests'),
    (4, dict(beam_width=2, eos_id=5, length_penalty=[1.0, 1.0, 1.0], early_stopping=[True] * 3),
     'length_penalty: 3 values for 4 requests'),
    (4, dict(beam_width=2, eos_id=5, early_stopping=[True] * 3), 'early_stopping: 3 values for 4 requests'),
    (4, dict(beam_width=2, eos_id=5, early_stopping=["sometimes"] * 3), 'early_stopping: 3 values for 4 requests'),
    (4, dict(beam_width=2, eos_id=5, early_stopping="sometimes"),
     'early_stopping must be False, True or "never" (got \'sometimes\')'),
    (4, dict(beam_width=2, eos_id=5, early_stopping=[False, True, "never", "sometimes"]),
     'early_stopping must be False, True or "never" (got \'sometimes\')'),
    (4, dict(beam_width=2, eos_id=5, length_penalty=[0.5, 1.0, 1.5, 2.0], early_stopping=[False, True, "never", True]), ACCEPTED),
    (4, dict(beam_width=2, length_penalty=[1.0], early_stopping="sometimes"), ACCEPTED),
    (4, dict(token_bitmask=True, logit_bias_capacity=16), ACCEPTED),
    (4, dict(token_bitmask=True, tp_size=2),
     'token_bitmask / logit_bias need tp_size 1 (got tp_size 2): the vocabulary-parallel argmax would need a mask '
     'sharded by vocabulary'),
    (4, dict(logit_bias_capacity=16, tp_size=2),
     'token_bitmask / logit_bias need tp_size 1 (got tp_size 2): the vocabulary-parallel argmax would need a mask '
     'sharded by vocabulary'),
    (4, dict(logit_bias_capacity=-1), 'logit_bias_capacity must be >= 0 (got -1)'),
    (4, dict(logit_bias_capacity=-1, tp_size=2), 'logit_bias_capacity must be >= 0 (got -1)'),
    (4, dict(token_bitmask=True, sampling=BAD_MINP, tp_size=2),
     'token_bitmask / logit_bias need tp_size 1 (got tp_size 2): the vocabulary-parallel argmax would need a mask '
     'sharded by vocabulary'),
    (129, dict(token_bitmask=True, tp_size=2),
     'token_bitmask / logit_bias need tp_size 1 (got tp_size 2): the vocabulary-parallel argmax would need a mask '
     'sharded by vocabulary'),
    (4, dict(token_bitmask=True, logit_bias_capacity=8, beam_width=2, eos_id=5), ACCEPTED),
    (4, dict(shared_prefix=(2, 16)), ACCEPTED),
    (4, dict(shared_prefix=(0, 16)), 'shared_prefix: (requests_per_prefix >= 1, prefix_tokens >= 0) (got (0, 16))'),
    (4, dict(shared_prefix=(2, -1)), 'shared_prefix: (requests_per_prefix >= 1, prefix_tokens >= 0) (got (2, -1))'),
    (4, dict(shared_prefix=(0, 16), q_len=2), 'shared_prefix: (requests_per_prefix >= 1, prefix_tokens >= 0) (got (0, 16))'),
    (4, dict(shared_prefix=(2, 16), q_len=2),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 2, '
     'tree False, beam_width 1, sampling False, tp_size 1)'),
    (4, dict(shared_prefix=(2, 16), q_len=3, tree=TREE),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 3, '
     'tree True, beam_width 1, sampling False, tp_size 1)'),
    (4, dict(shared_prefix=(2, 16), beam_width=2),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 1, '
     'tree False, beam_width 2, sampling False, tp_size 1)'),
    (4, dict(shared_prefix=(2, 16), sampling=SP),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 1, '
     'tree False, beam_width 1, sampling True, tp_size 1)'),
    (4, dict(shared_prefix=(2, 16), tp_size=2),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 1, '
     'tree False, beam_width 1, sampling False, tp_size 2)'),
    (4, dict(shared_prefix=(2, 16), beam_width=2, logit_bias_capacity=-1),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 1, '
     'tree False, beam_width 2, sampling False, tp_size 1)'),
    (4, dict(shared_prefix=(2, 16), token_bitmask=True, tp_size=2),
     'shared_prefix needs the greedy step: q_len 1, no tree, beam_width 1, no sampling and tp_size 1 (got q_len 1, '
     'tree False, beam_width 1, sampling False, tp_size 2)'),
    (4, dict(shared_prefix=(2, 16), token_bitmask=True), ACCEPTED),
    (257, dict(shared_prefix=(2, 16)),
     'a step runs at most 256 token rows (the GEMM row limit), and at most 128 with tp_size > 1 (got 257 rows, tp_size'
     ' 1)'),
    (4, dict(act_order=True), ACCEPTED),
    (4, dict(act_order=True, cfg=F16), 'act_order needs tp_size 1 and quant int4 / int8g (got tp_size 1, quant f16)'),
    (4, dict(act_order=True, tp_size=2), 'act_order needs tp_size 1 and quant int4 / int8g (got tp_size 2, quant int4)'),
    (257, dict(act_order=True, tp_size=2),
     'a step runs at most 256 token rows (the GEMM row limit), and at most 128 with tp_size > 1 (got 257 rows, tp_size'
     ' 2)'),
    (4, dict(act_order=True, q_len=2, tree=TREE, sampling=SP, token_bitmask=True), ACCEPTED),
]


def _outcome(batch, cfg=TINY, **options) -> str:
    try:
        DecodeStep(cfg, batch, 40, torch.device("cpu"), **options)
    except ValueError as e:
        return str(e)
    except B200Error as e:
        assert "expected contiguous CUDA tensors" in str(e), e
        return ACCEPTED
    raise AssertionError("a DecodeStep on the CPU got past its weight packing")


def test_each_option_set_gets_its_first_message():
    wrong = [(batch, options, got, want) for batch, options, want in CASES
             if (got := _outcome(batch, **options)) != want]
    assert not wrong, "\n".join(f"batch {b} {o}: got {g!r}, want {w!r}" for b, o, g, w in wrong)


def test_sampling_parameter_counts_are_checked_last_before_any_allocation():
    """A per-request sampling parameter of the wrong length is refused with the other options, after all of them; a parameter
    the step does not upload (penalties all off, min_p all 0) is not counted."""
    cpu = torch.device("cpu")
    for sp in (SamplingParams(temperature=[1.0] * 3), SamplingParams(top_k=[5] * 5), SamplingParams(top_p=(0.9,)),
               SamplingParams(frequency=[0.1] * 3), SamplingParams(min_p=[0.1] * 3)):
        with pytest.raises(ValueError, match=r"^sampling: \d values for 4 requests$"):
            DecodeStep(TINY, 4, 40, cpu, sampling=sp)
    with pytest.raises(ValueError, match="act_order needs"):
        DecodeStep(F16, 4, 40, cpu, sampling=SamplingParams(temperature=[1.0] * 3), act_order=True)
    for sp in (SamplingParams(repetition=[1.0] * 3), SamplingParams(min_p=[0.0] * 3)):
        with pytest.raises(B200Error, match="expected contiguous CUDA tensors"):
            DecodeStep(TINY, 4, 40, cpu, sampling=sp)
