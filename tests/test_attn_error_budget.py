"""CPU self-test of the attention error budget (oracle.attn_error_budget) that the GPU parity tests check the kernel with:
at the full-size decode shapes it must accept the C oracle, which rounds P to the cache type as the kernel does, and it
must reject references that lost a token, a tile or a split. No GPU needed."""
import numpy as np
import pytest

from oracle import oracle as orc

FULL = [("Llama-3-8B B32 S2048", 32, 32, 8, 2048), ("Qwen2-72B TP8 B16 S8192", 16, 8, 1, 8192)]
T, D = 64, 128


def _case(B, Hq, Hkv, S, is_bf16, seed=0):
    rng = np.random.default_rng(seed)
    npages = B * S // T + 1
    pool = orc.to_bits(rng.standard_normal((npages, 2, Hkv, T, D), dtype=np.float32), is_bf16)
    q = orc.to_bits(rng.standard_normal((B, Hq, D), dtype=np.float32), is_bf16)
    block_ids = (rng.permutation(npages - 1) + 1).astype(np.int32).reshape(B, S // T)
    seq = np.full(B, S - 1, np.int32)
    return q, pool, block_ids, seq


@pytest.mark.parametrize("is_bf16", [False, True], ids=["fp16", "bf16"])
@pytest.mark.parametrize("cfg", FULL, ids=[c[0] for c in FULL])
def test_attn_error_budget_accepts_the_oracle_and_rejects_lost_tokens(cfg, is_bf16):
    name, B, Hq, Hkv, S = cfg
    q, pool, block_ids, seq = _case(B, Hq, Hkv, S, is_bf16)
    qf, poolf = orc.from_bits(q, is_bf16), orc.from_bits(pool, is_bf16)
    ref, E = orc.paged_decode_attn_np(qf, poolf, block_ids, seq, T, with_abs=True)
    budget = orc.attn_error_budget(ref, E, is_bf16)
    got = orc.from_bits(orc.paged_decode_attn(q, pool, orc.convert_block_table(block_ids), seq, Hq, Hkv, D, T,
                                              is_bf16=is_bf16), is_bf16)
    worst = float((np.abs(got - ref) / budget).max())
    print(f"{name} {'bf16' if is_bf16 else 'fp16'}: C oracle worst err/budget {worst:.3f}")
    assert worst <= 1.0

    # The op has no positional term, so a reference that lost positions is the same op on fewer pages.
    half = S // 2 // T
    mutants = {"tile 64..127 dropped": (np.delete(block_ids, 1, axis=1), seq - T),
               "first half dropped": (np.ascontiguousarray(block_ids[:, half:]), seq - half * T)}
    if not (is_bf16 and S == 8192):
        # bf16 at 8192 tokens: one token moves the output by less than the budget; the exact position probes of the GPU
        # suite (uniform scores, dominant key) catch a dropped last token at any length instead
        mutants["last token dropped"] = (block_ids, seq - 1)
    for what, (bid, sq) in mutants.items():
        mut = orc.paged_decode_attn_np(qf, poolf, bid, sq, T)
        nbad = int((np.abs(mut - ref) > budget).sum())
        print(f"  {what}: {nbad}/{ref.size} elements over budget")
        assert nbad > 0, what
