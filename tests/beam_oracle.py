"""Float64 numpy reference of one beam-search step (b200_beam_search_step) and of the no-repeat-n-gram ban
(b200_ban_repeat_ngram), restated from the Hugging Face / TensorRT-LLM beam-search convention."""
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
