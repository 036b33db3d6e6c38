"""Float64 numpy reference of b200_token_logprobs: the log-softmax of each row of logits as given, the drawn token's value
and the top n by value descending, equal values by lower id."""
import numpy as np


def log_softmax_np(logits):
    """[rows, V] float64 log-softmax; NaN counts as -inf, a row without a finite logit gives NaN."""
    x = np.asarray(logits, np.float64)
    x = np.where(np.isnan(x), -np.inf, x)
    m = x.max(axis=-1, keepdims=True)
    finite = np.isfinite(m)
    mm = np.where(finite, m, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        lse = mm + np.log(np.exp(x - mm).sum(axis=-1, keepdims=True))
        lp = x - lse
    return np.where(finite, lp, np.nan)


def token_logprobs_np(logits, top_n, tokens=None):
    """Returns dict(lp [rows, V]; top_ids / top_logprobs [rows, top_n]; ranked [rows, top_n + 1]: the values of the first top_n + 1
    ranks, for gap checks at the cutoff; token_logprob [rows] when tokens is given, NaN for an id outside [0, V))."""
    lp = log_softmax_np(logits)
    rows, V = lp.shape
    key = np.where(np.isnan(lp), -np.inf, lp)
    ids = np.arange(V)
    order = np.stack([np.lexsort((ids, -key[r]))[: top_n + 1] for r in range(rows)]) if rows else np.zeros((0, top_n + 1), int)
    out = dict(lp=lp, top_ids=order[:, :top_n], top_logprobs=np.take_along_axis(lp, order[:, :top_n], 1),
               ranked=np.take_along_axis(lp, order, 1))
    if tokens is not None:
        t = np.asarray(tokens, np.int64)
        ok = (t >= 0) & (t < V)
        out["token_logprob"] = np.where(ok, lp[np.arange(rows), np.clip(t, 0, V - 1)], np.nan)
    return out
