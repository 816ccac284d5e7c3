"""Float64 numpy restatement of MCD-DTW (DESIGN.md section 8h; the device form is kernels_mcd.cu).  Test aid only: the
product never imports it.

Per frame of dB-normalised mels x (n_mels,): a = (ln 10 / 20) (max_db x - max_db + ref_db), c = D[1:K+1] a with D the
orthonormal DCT-II matrix.  Local cost d(i, j) = (10 / ln 10) sqrt(2 sum_k (cx_ik - cy_jk)^2).  D(0, 0) = d(0, 0),
D(i, j) = d(i, j) + min(D(i-1, j-1), D(i-1, j), D(i, j-1)), a tie going to the first of the three; the path ends at
(nx - 1, ny - 1); mcd = D_end / P with P the cells on the path."""
import numpy as np

LN10_20 = np.log(10.0) / 20.0
COST_SCALE = 10.0 / np.log(10.0)


def dct_matrix(M):
    """The orthonormal DCT-II matrix (M, M): D[k, m] = sqrt((1 if k == 0 else 2) / M) cos(pi k (2m + 1) / (2M))."""
    k = np.arange(M, dtype=np.float64)[:, None]
    m = np.arange(M, dtype=np.float64)[None, :]
    D = np.sqrt(2.0 / M) * np.cos(np.pi * k * (2 * m + 1) / (2.0 * M))
    D[0] /= np.sqrt(2.0)
    return D


def cepstrum(mels, K, max_db=100.0, ref_db=20.0):
    """(T, n_mels) dB-normalised mels -> (T, K) float64 coefficients 1 .. K."""
    x = np.asarray(mels, np.float32).astype(np.float64)
    a = LN10_20 * (max_db * x - max_db + ref_db)
    return a @ dct_matrix(x.shape[1])[1:K + 1].T


def local_cost(cx, cy):
    """(nx, K), (ny, K) -> (nx, ny) d(i, j)."""
    out = np.empty((cx.shape[0], cy.shape[0]))
    for i in range(0, cx.shape[0], 128):                # in row blocks: long sequences stay within memory
        diff = cx[i:i + 128, None, :] - cy[None, :, :]
        out[i:i + 128] = COST_SCALE * np.sqrt(2.0 * (diff * diff).sum(-1))
    return out


def dtw(d):
    """The DTW of a cost matrix d (nx, ny) -> dict(path (P, 2) int64 from (0, 0), total D_end, pairs P, mcd, margin).
    `margin` is the smallest gap between the chosen predecessor and the runner-up over the cells of the path (inf where a
    cell has one predecessor): below about 1e-9 relative, a last-bit difference in the costs may choose another path."""
    d = np.asarray(d, np.float64)
    nx, ny = d.shape
    D = np.full((nx, ny), np.inf)
    bp = np.zeros((nx, ny), np.int64)
    gap = np.full((nx, ny), np.inf)
    for s in range(nx + ny - 1):                    # anti-diagonals, as the device sweeps them
        i = np.arange(max(0, s - (ny - 1)), min(s, nx - 1) + 1)
        j = s - i
        if s == 0:
            D[0, 0] = d[0, 0]
            continue
        cand = np.full((len(i), 3), np.inf)
        m = (i > 0) & (j > 0)
        cand[m, 0] = D[i[m] - 1, j[m] - 1]
        m = i > 0
        cand[m, 1] = D[i[m] - 1, j[m]]
        m = j > 0
        cand[m, 2] = D[i[m], j[m] - 1]
        c = np.argmin(cand, axis=1)                 # the first minimum: diagonal, then advance X, then advance Y
        best = cand[np.arange(len(i)), c]
        runner = np.sort(cand, axis=1)[:, 1]
        gap[i, j] = np.where(np.isfinite(runner), runner - best, np.inf)
        D[i, j] = d[i, j] + best
        bp[i, j] = c
    i, j = nx - 1, ny - 1
    path = [(i, j)]
    while (i, j) != (0, 0):
        c = bp[i, j]
        i, j = i - (c != 2), j - (c != 1)
        path.append((i, j))
    path = np.array(path[::-1], np.int64)
    P = len(path)
    margin = float(gap[path[1:, 0], path[1:, 1]].min()) if P > 1 else np.inf
    total = float(D[-1, -1])
    return dict(path=path, total=total, pairs=P, mcd=total / P, margin=margin)


def mcd_dtw(x, y, K=24, max_db=100.0, ref_db=20.0):
    """MCD-DTW of one pair of mel sequences (nx, n_mels), (ny, n_mels)."""
    return dtw(local_cost(cepstrum(x, K, max_db, ref_db), cepstrum(y, K, max_db, ref_db)))


def mcd_batch(X, nx, Y, ny, K=24, max_db=100.0, ref_db=20.0):
    """X (B, Tx, n_mels), Y (B, Ty, n_mels) -> padded outputs as dctts_mcd_dtw writes them: mcd (B,), pairs (B,),
    path (B, Tx + Ty - 1, 2) with -1 past pairs[b], and margin (B,)."""
    X, Y = np.asarray(X), np.asarray(Y)
    B, Tx, Ty = X.shape[0], X.shape[1], Y.shape[1]
    out = dict(mcd=np.zeros(B), pairs=np.zeros(B, np.int64), path=np.full((B, Tx + Ty - 1, 2), -1, np.int64),
               margin=np.zeros(B))
    for b in range(B):
        r = mcd_dtw(X[b, :int(nx[b])], Y[b, :int(ny[b])], K, max_db, ref_db)
        out["mcd"][b], out["pairs"][b], out["margin"][b] = r["mcd"], r["pairs"], r["margin"]
        out["path"][b, :r["pairs"]] = r["path"]
    return out


def window_checks(P, n, e, t, max_T):
    """The free run's window checks for one utterance: P (>= n,) the window of every frame, n frames run, e the EOS
    position, t the recording's frames.  Returns dict(eos_reached, skipped, longest_stall, length_ratio)."""
    P = np.asarray(P[:n], np.int64)
    skipped = int(e - np.isin(np.arange(e), P).sum()) if e > 0 else 0
    runs, best = 1, 1
    for k in range(1, n):
        runs = runs + 1 if P[k] == P[k - 1] else 1
        best = max(best, runs)
    return dict(eos_reached=bool(n < max_T), skipped=skipped, longest_stall=best if n > 0 else 0,
                length_ratio=n / float(t))
