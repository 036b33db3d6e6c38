"""GPU tests of how a decode program keeps the launches that run outside its persistent kernel.

One program holds every such entry point: the four attention entries, an FP16 GEMM, a norm too wide for the persistent
kernel, qk_rmsnorm, silu_and_mul, permute_cols, rope_append_ex, argmax, sample, spec_verify, the beam step, both
beam-hypothesis kernels, token_logprobs and the n-gram ban. Everything a call decides is decided when it is recorded: a
launch of the program gives the bits of the same calls made eagerly, after the caller has overwritten the b200_rope_config
it passed, and after a test-hook variable that forced a launch plan while recording is unset."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import RopeConfig  # noqa: E402

DEV = torch.device("cuda:0")
B, HQ, HKV, D, T, M = 2, 8, 2, 128, 16, 64      # sequences, heads, head_dim, page size, pages per sequence
MAX_LEN = T * M
W, V, HIST, MAX_HYP = 2, 1000, 12, 16           # beam width, vocabulary, history stride, hypothesis length
EOS = 7
RB, K, N = 4, 4096, 256                         # rows of the glue ops, the FP16 GEMM's K and N
WIDE = 9216                                     # add_rmsnorm wider than the persistent kernel's norm (8192): its own launch
FORCED = {"B200_ATTN_TILES_PER_SPLIT": "16", "B200_GEMM_SPLITK": "1"}   # one split each; the plans pick more here


class Case:
    """Seeded inputs and zeroed outputs of every call, in one dict of device tensors that reset() restores."""

    def __init__(self, seed=0):
        g = torch.Generator().manual_seed(seed)
        h, f32, i32 = torch.float16, torch.float32, torch.int32

        def rnd(*shape, dtype=h, scale=1.0):
            return (torch.randn(*shape, generator=g) * scale).to(dtype)

        def ints(hi, *shape):
            return torch.randint(0, hi, shape, generator=g, dtype=i32)

        qkv_n = (HQ + 2 * HKV) * D
        beam_logits = rnd(B * W, V, dtype=f32)
        beam_logits[::2, EOS] += 6.0                 # EOS among the best candidates of some beams
        t = dict(
            pool=rnd(1 + B * M, 2, HKV, T, D), block_ids=(torch.randperm(B * M, generator=g) + 1).to(i32).view(B, M),
            seq=torch.tensor([700, 950], dtype=i32), shared=torch.zeros(1, dtype=i32),
            q=rnd(B, HQ, D), q_multi=rnd(B, 2, HQ, D), q_beam=rnd(1, W, HQ, D), qkv_rope=rnd(B, qkv_n),
            attn=torch.zeros(B, HQ * D, dtype=h), attn_multi=torch.zeros(B, 2, HQ * D, dtype=h),
            attn_beam=torch.zeros(1, W, HQ * D, dtype=h), attn_rope=torch.zeros(B, HQ * D, dtype=h),
            gx=rnd(RB, K), gw=rnd(K, N, scale=0.02), gy=torch.zeros(RB, N, dtype=h),
            wide_x=rnd(RB, WIDE), wide_res=rnd(RB, WIDE), wide_g=rnd(WIDE), wide_y=torch.zeros(RB, WIDE, dtype=h),
            qkv_norm=rnd(B, qkv_n), q_gamma=rnd(D), k_gamma=rnd(D),
            gate_up=rnd(RB, 1024), act=torch.zeros(RB, 512, dtype=h),
            px=rnd(RB, 1024), perm=torch.randperm(1024, generator=g).to(i32), py=torch.zeros(RB, 1024, dtype=h),
            qkv_ex=rnd(B, qkv_n), q_ex=torch.zeros(B, HQ * D, dtype=h),
            am_logits=rnd(RB, V), am_out=torch.zeros(RB, dtype=i32),
            s_logits=rnd(RB, V, dtype=f32), top_k=torch.tensor([0, 5, 50, 1], dtype=i32),
            top_p=torch.tensor([1.0, 0.9, 0.8, 1.0]), uniform=torch.rand(RB, generator=g),
            temperature=torch.tensor([1.0, 0.7, 1.3, 1.0]), s_token=torch.zeros(RB, dtype=i32), s_prob=torch.zeros(RB),
            drafts=ints(4, B, 2), target_ids=ints(4, B, 3), sv_tokens=torch.zeros(B, 3, dtype=i32),
            sv_accepted=torch.zeros(B, dtype=i32),
            beam_logits=beam_logits, beam_cum=rnd(B, W, dtype=f32), beam_ws=ops.beam_search_workspace(B, W, V, "cpu"),
            history=ints(5, B * W, HIST), hist_len=torch.tensor([HIST, 3, 0, 9], dtype=i32),
            length_penalty=torch.tensor([1.0, 0.5]), early_stopping=torch.tensor([0, 1], dtype=i32),
            hyp_state=ops.beam_hypotheses_state(B, W, MAX_HYP, "cpu"), hyp_done=torch.zeros(B, dtype=i32),
            lp_logits=rnd(RB, V), lp_tokens=ints(V, RB), lp_ws=ops.token_logprobs_workspace(RB, V, 5, "cpu"),
            ban_logits=rnd(RB, V, dtype=f32), ngram=torch.tensor([2, 3, 0, 2], dtype=i32))
        for k, (dt, shape) in dict(cand_token=(i32, (B, 2 * W)), cand_parent=(i32, (B, 2 * W)), cand_score=(f32, (B, 2 * W)),
                                   next_token=(i32, (B, W)), next_parent=(i32, (B, W)), next_cum=(f32, (B, W)),
                                   fin_tokens=(i32, (B, W, MAX_HYP)), fin_len=(i32, (B, W)), fin_score=(f32, (B, W)),
                                   fin_cum=(f32, (B, W)), lp_top_ids=(i32, (RB, 5)), lp_top=(f32, (RB, 5)),
                                   lp_token=(f32, (RB,))).items():
            t[k] = torch.zeros(shape, dtype=dt)
        self.t = {k: v.to(DEV) for k, v in t.items()}
        self.init = {k: v.clone() for k, v in self.t.items()}
        self.page_list = ops.convert_block_table(self.t["block_ids"])
        self.attn_ws = ops.attn_workspace(B, HQ, HKV, MAX_LEN, DEV)
        self.gemm_ws = ops.gemm_workspace(RB, [(K, N)], DEV)
        self.gw = ops.pack_f16(self.t["gw"])
        self.rope = RopeConfig(style=1, dim=D, base=10000.0, scale=1.0, max_pos=0, extrapolation_factor=1.0, mscale=1.0)

    def calls(self):
        """The program's calls: each one is its own launch inside a program, none is an op of the persistent kernel."""
        t, pl, ws = self.t, self.page_list, self.attn_ws
        ops.paged_decode_attn(t["q"], t["pool"], pl, t["seq"], MAX_LEN, ws, out=t["attn"])
        ops.paged_decode_attn_multi(t["q_multi"], t["pool"], pl, t["seq"], MAX_LEN, ws, out=t["attn_multi"])
        ops.paged_decode_attn_beam(t["q_beam"], t["pool"], pl, t["seq"], t["shared"], MAX_LEN, ws, out=t["attn_beam"])
        ops.paged_decode_attn_rope(t["qkv_rope"], t["pool"], pl, t["seq"], HQ, MAX_LEN, 10000.0, ws, out=t["attn_rope"])
        ops.wo_gemm(t["gx"], self.gw, self.gemm_ws, out=t["gy"])
        ops.add_rmsnorm(t["wide_x"], t["wide_res"], t["wide_g"], 1e-5, out=t["wide_y"])
        ops.qk_rmsnorm(t["qkv_norm"], t["q_gamma"], t["k_gamma"], HQ, HKV, D, 1e-6)
        ops.silu_and_mul(t["gate_up"], out=t["act"])
        ops.permute_cols(t["px"], t["perm"], out=t["py"])
        ops.rope_append_ex(t["qkv_ex"], t["pool"], pl, t["seq"], HQ, self.rope, q_out=t["q_ex"])
        ops.argmax(t["am_logits"], out=t["am_out"])
        ops.sample(t["s_logits"], t["top_k"], t["top_p"], t["uniform"], temperature=t["temperature"],
                   out=dict(token=t["s_token"], token_prob=t["s_prob"]))
        ops.spec_verify(t["drafts"], target_ids=t["target_ids"], out_tokens=t["sv_tokens"], accepted=t["sv_accepted"])
        beam = ops.beam_search_step(t["beam_logits"], t["beam_cum"], W, EOS, workspace=t["beam_ws"],
                                    out={k: t[k] for k in ("cand_token", "cand_parent", "cand_score", "next_token", "next_parent",
                                                           "next_cum")})
        ops.beam_hypotheses_update(beam, t["history"], t["hist_len"], EOS, t["length_penalty"], t["early_stopping"], t["hyp_state"],
                                   t["hyp_done"], MAX_HYP)
        ops.beam_hypotheses_finalize(t["hyp_state"], t["hyp_done"], t["next_cum"], t["history"], t["hist_len"], W, MAX_HYP,
                                     t["length_penalty"], out=dict(tokens=t["fin_tokens"], len=t["fin_len"], score=t["fin_score"],
                                                                   cum=t["fin_cum"]))
        ops.token_logprobs(t["lp_logits"], 5, t["lp_tokens"], workspace=t["lp_ws"],
                           out=dict(top_ids=t["lp_top_ids"], top_logprobs=t["lp_top"], token_logprob=t["lp_token"]))
        ops.ban_repeat_ngram(t["ban_logits"], t["history"], t["hist_len"], t["ngram"])

    CALLS = 18

    def reset(self):
        for k, v in self.t.items():
            v.copy_(self.init[k])

    def snapshot(self):
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in self.t.items()}

    def eager(self):
        self.reset()
        self.calls()
        return self.snapshot()

    def launch(self, prog):
        self.reset()
        prog.launch()
        return self.snapshot()


def differing(a, b):
    """Names of the tensors whose bits differ."""
    return sorted(k for k in a if not torch.equal(a[k].view(torch.uint8), b[k].view(torch.uint8)))


def test_launches_give_the_eager_bits_after_the_callers_rope_config_changes():
    case = Case()
    eager = case.eager()
    prog = ops.Program()
    n0 = ops.launch_count()
    with prog.record():
        case.calls()
    assert ops.launch_count() == n0, "recording launched a kernel"
    assert prog.num_ops == 0 and prog.num_launches == Case.CALLS
    case.rope.base, case.rope.dim = 500000.0, 64     # the caller reuses its b200_rope_config after the call
    for _ in range(2):
        n0 = ops.launch_count()
        got = case.launch(prog)
        assert ops.launch_count() - n0 == prog.num_launches
        assert not differing(got, eager)
    assert "q_ex" in differing(case.eager(), eager), "the overwritten config computes something else eagerly"


def test_a_plan_forced_while_recording_is_kept_after_the_variable_is_unset(monkeypatch):
    case = Case(seed=1)
    default = case.eager()
    for k, v in FORCED.items():
        monkeypatch.setenv(k, v)
    forced = case.eager()
    assert {"attn", "attn_multi", "attn_beam", "attn_rope", "gy"} <= set(differing(forced, default)), "the forced plans change no bits"
    prog = ops.Program()
    with prog.record():
        case.calls()
    for k in FORCED:
        monkeypatch.delenv(k)
    assert not differing(case.launch(prog), forced)
