"""Float64 numpy reference of one beam-search step (b200_beam_search_step) and of the no-repeat-n-gram ban
(b200_ban_repeat_ngram), restated from the Hugging Face / TensorRT-LLM beam-search convention, and the pass rule of a kernel's
selection against it (check_beam)."""
import numpy as np


def beam_scores_np(logits, cum):
    """Scores [B, W, V] in float64: cum[b][i] + log_softmax(row b*W + i)[v]. -inf logits, rows with cum -inf and rows without
    a finite logit give -inf. NaN logits count as -inf, as in the kernel."""
    cum = np.asarray(cum, np.float64)
    B, W = cum.shape
    x = np.asarray(logits, np.float64).reshape(B, W, -1)
    x = np.where(np.isnan(x), -np.inf, x)
    m = x.max(axis=-1, keepdims=True)
    finite_m = np.where(np.isfinite(m), m, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        lse = finite_m + np.log(np.exp(x - finite_m).sum(axis=-1, keepdims=True))
        s = cum[..., None] + (x - lse)
    dead = ~(cum > -np.inf)[..., None] | ~np.isfinite(x)
    return np.where(dead, -np.inf, s)


def beam_step_np(logits, cum, eos_id=-1):
    """The beam step on logits [B*W, V] and cum [B, W]. Returns dict of cand_token / cand_parent / cand_score [B, 2W] (ranked by
    score descending, then by lower flat index i*V + v), next_token / next_parent / next_cum [B, W] (the first W candidates that
    are not eos_id), and ranked_scores [B, 2W + 1] (the scores of the first 2W + 1 ranks, for gap checks at the cutoff)."""
    cum = np.asarray(cum, np.float64)
    B, W = cum.shape
    s = beam_scores_np(logits, cum).reshape(B, -1)
    V = s.shape[1] // W
    flat = np.arange(W * V)
    out = {k: [] for k in ("cand_token", "cand_parent", "cand_score", "next_token", "next_parent", "next_cum", "ranked_scores")}
    for b in range(B):
        order = np.lexsort((flat, -s[b]))[: 2 * W + 1]      # -(-inf) = +inf sorts last, ties by index
        top = order[: 2 * W]
        out["cand_token"].append(top % V)
        out["cand_parent"].append(top // V)
        out["cand_score"].append(s[b, top])
        out["ranked_scores"].append(s[b, order])
        keep = top[top % V != eos_id][:W]
        out["next_token"].append(keep % V)
        out["next_parent"].append(keep // V)
        out["next_cum"].append(s[b, keep])
    return {k: np.stack(v) for k, v in out.items()}


def next_from_candidates(cand_token, cand_parent, cand_score, W, eos_id=-1):
    """The EOS rule on ranked candidates [B, 2W]: the first W whose token is not eos_id."""
    keep = [np.nonzero(cand_token[b] != eos_id)[0][:W] for b in range(cand_token.shape[0])]
    return (np.stack([cand_token[b, k] for b, k in enumerate(keep)]), np.stack([cand_parent[b, k] for b, k in enumerate(keep)]),
            np.stack([cand_score[b, k] for b, k in enumerate(keep)]))


def score_tol(score):
    return 1e-5 * (1.0 + np.abs(score))


def check_beam(got, exp, W, eos_id):
    """The pass rule against the float64 reference: scores within 1e-5 * (1 + |score|) rank by rank; tokens and parents
    equal at every rank whose reference score is clear of its neighbours by that bound (or exactly tied, which both rank by
    flat index); the next_* arrays follow from the kernel's own candidates by the EOS rule exactly."""
    es, rs = exp["cand_score"], exp["ranked_scores"]
    gs = got["cand_score"].astype(np.float64)
    fin = np.isfinite(es)
    assert (np.isneginf(gs) == np.isneginf(es)).all(), (gs, es)
    assert (np.abs(gs[fin] - es[fin]) <= score_tol(es[fin])).all(), np.abs(gs - es)[fin].max()
    B = es.shape[0]
    for b in range(B):
        for r in range(2 * W):
            def clear(a, c):
                if np.isneginf(a) and np.isneginf(c):
                    return True                                  # both -inf: an exact tie, ranked by index
                d = abs(a - c)
                return d == 0 or d > score_tol(a)
            ok = clear(rs[b, r], rs[b, r + 1]) and (r == 0 or clear(rs[b, r - 1], rs[b, r]))
            tied = (r > 0 and rs[b, r - 1] == rs[b, r]) or rs[b, r] == rs[b, r + 1]
            if ok or tied and np.isneginf(rs[b, r]):
                assert got["cand_token"][b, r] == exp["cand_token"][b, r], (b, r, got["cand_token"][b], exp["cand_token"][b])
                assert got["cand_parent"][b, r] == exp["cand_parent"][b, r], (b, r)
    nt, npar, nc = next_from_candidates(got["cand_token"], got["cand_parent"], got["cand_score"], W, eos_id)
    np.testing.assert_array_equal(got["next_token"], nt)
    np.testing.assert_array_equal(got["next_parent"], npar)
    np.testing.assert_array_equal(got["next_cum"], nc)


def banned_np(history, hist_len, ngram_size, vocab):
    """Per row, the sorted token ids the no-repeat-n-gram rule bans: for n = ngram_size[r] > 0 and L = min(hist_len[r], stride),
    every start s in [0, L - n] with h[s .. s+n-2] == h[L-n+1 .. L-1] bans h[s+n-1]; ids outside [0, vocab) are ignored."""
    history = np.asarray(history)
    out = []
    for r in range(history.shape[0]):
        n, L = int(ngram_size[r]), min(int(hist_len[r]), history.shape[1])
        h = history[r, :L]
        ban = set()
        if n > 0:
            suffix = h[L - n + 1:] if n > 1 else h[:0]
            for s in range(0, L - n + 1):
                if np.array_equal(h[s:s + n - 1], suffix):
                    t = int(h[s + n - 1])
                    if 0 <= t < vocab:
                        ban.add(t)
        out.append(np.array(sorted(ban), dtype=np.int64))
    return out
