"""Float64 numpy restatement of the aligner's search (DESIGN.md section 4d; the device form is kernels_align.cu).  Test
aid only: the product never imports it.

The best path through A (N, T) for T_b frames ending at the text end e, with window size w: one character n_t per
frame, 0 <= n_0 <= w - 1, 0 <= n_t - n_{t-1} <= w - 1, n_{T_b - 1} = e, maximising the sum of
c[n, t] = log(double(max(A[n, t], 1e-30f))) added in frame order; of two equal predecessors the smaller step wins."""
import numpy as np


def cost(A):
    """c = log(double(max(A, 1e-30f))): the floor in float32, the log in float64."""
    return np.log(np.maximum(np.asarray(A, np.float32), np.float32(1e-30)).astype(np.float64))


def band(t, T_b, e, w):
    """The cells of frame t that can be reached and can still reach e: [lo, hi]."""
    return max(0, e - (w - 1) * (T_b - 1 - t)), min(e, (w - 1) * (t + 1))


def search(A, T_b, e, w):
    """A (N, >= T_b) -> dict(chars (T_b,), path (T_b,), durations (N,), score, margin).  `margin` is the smallest gap, in
    D, between the best predecessor and the runner-up over the cells of the returned path (inf where a cell has one
    predecessor): below about 1e-9 a last-bit difference in the costs may choose another path."""
    N = A.shape[0]
    if not (1 <= T_b <= A.shape[1] and 0 <= e < N and e <= (w - 1) * T_b):
        raise ValueError("search: T_b %d, e %d, w %d are not admissible for A %s" % (T_b, e, w, A.shape))
    c = cost(A[:, :T_b])
    D = np.full(e + 1, -np.inf)
    lo, hi = band(0, T_b, e, w)
    D[lo:hi + 1] = c[lo:hi + 1, 0]
    bp = np.zeros((T_b, e + 1), np.int64)
    gap = np.full((T_b, e + 1), np.inf)
    for t in range(1, T_b):
        lo, hi = band(t, T_b, e, w)
        plo, phi = band(t - 1, T_b, e, w)
        n = np.arange(lo, hi + 1)
        src = n[:, None] - np.arange(w)[None, :]                       # (cells, w): the predecessor of step s
        ok = (src >= plo) & (src <= phi)
        cand = np.where(ok, D[np.clip(src, 0, e)], -np.inf)
        s = np.argmax(cand, axis=1)                                    # the first maximum: the smaller step
        best = cand[np.arange(len(n)), s]
        if w > 1:
            runner = np.sort(cand, axis=1)[:, -2]
            gap[t, lo:hi + 1] = np.where(np.isfinite(runner), best - runner, np.inf)
        Dn = np.full(e + 1, -np.inf)
        Dn[lo:hi + 1] = c[lo:hi + 1, t] + best
        bp[t, lo:hi + 1] = s
        D = Dn
    chars = np.empty(T_b, np.int64)
    chars[-1] = e
    for t in range(T_b - 1, 0, -1):
        chars[t - 1] = chars[t] - bp[t, chars[t]]
    path = np.concatenate([[0], chars[:-1]])
    durations = np.bincount(chars, minlength=N)
    margin = float(gap[np.arange(1, T_b), chars[1:]].min()) if T_b > 1 else np.inf
    return dict(chars=chars, path=path, durations=durations, score=float(D[e]), margin=margin)


def path_score(A, chars):
    """The summed cost of a path in the search's order of additions (c[n_t, t] + the sum over the earlier frames)."""
    c = cost(A)
    s = c[chars[0], 0]
    for t in range(1, len(chars)):
        s = c[chars[t], t] + s
    return float(s)


def admissible(chars, e, w):
    """Whether `chars` is a path the search may return for text end e and window size w."""
    ch = np.asarray(chars)
    d = np.diff(ch)
    return bool(0 <= ch[0] <= w - 1 and ch[-1] == e and ((d >= 0) & (d <= w - 1)).all())


def search_batch(A, lengths, ends, w):
    """A (B, N, T) -> padded outputs as dctts_align_search writes them: chars, path (B, T) with -1 past T_b, durations
    (B, N), score (B,), margin (B,)."""
    B, N, T = A.shape
    out = dict(chars=np.full((B, T), -1, np.int64), path=np.full((B, T), -1, np.int64),
               durations=np.zeros((B, N), np.int64), score=np.zeros(B), margin=np.zeros(B))
    for b in range(B):
        r = search(A[b], int(lengths[b]), int(ends[b]), w)
        k = int(lengths[b])
        out["chars"][b, :k], out["path"][b, :k] = r["chars"], r["path"]
        out["durations"][b], out["score"][b], out["margin"][b] = r["durations"], r["score"], r["margin"]
    return out
