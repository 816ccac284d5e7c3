"""Float64 restatement of a synthesis stream's grid (include/dctts.h: dctts_synth_stream_*, DESIGN.md section 8j).

Utterance b of `length` mel frames is committed in chunks of `chunk` frames, the last one ending at its length.  Chunk
[a, e) is one SSRN window, mel rows [max(0, a - left), min(length, e + right)), of which the magnitude rows
[r a, r e) are committed, and one vocoder push of those r (e - a) rows, final on the last chunk."""
import numpy as np

from dc_tts_b200.arch import ssrn_layers
from oracle import ref_numpy as rn


def halo(layers=None):
    """(left, right) mel frames of context for a run of committed frames: an output interval at the final rate walked
    back through the layer table (SAME taps [t - left, t + right], transposed conv output 2t reading x[t], x[t - 1])."""
    layers = ssrn_layers() if layers is None else layers
    up = 2 ** sum(l.kind == "D" for l in layers)
    a = 1000
    lo, hi = a * up, (a + 1) * up
    for l in reversed(layers):
        if l.kind == "D":
            lo, hi = (lo // 2 - 1 if lo % 2 == 0 else lo // 2), (hi - 1) // 2 + 1
        else:
            tot = (l.size - 1) * l.rate
            lft = tot if l.pad.lower() == "causal" else tot // 2
            lo, hi = lo - lft, hi + tot - lft
    return a - lo, hi - (a + 1)


def chunks(length, chunk, left, right):
    """The grid of one utterance: (a, e, s, t, final) per chunk -- committed mel rows [a, e), window rows [s, t)."""
    out = []
    for a in range(0, length, chunk):
        e = min(length, a + chunk)
        out.append((a, e, max(0, a - left), min(length, e + right), e == length))
    return out


def pushes(length, chunk, r=4):
    """The vocoder pushes of one utterance: (magnitude rows, final) per chunk."""
    return [(r * (e - a), fin) for a, e, _, _, fin in chunks(length, chunk, 0, 0)]


def ready_frames(length, chunk, right, k):
    """The published frame count at which chunk k is ready once the length is known."""
    return min(length, (k + 1) * chunk + right)


def ssrn64(P, Y):
    """float64 SSRN sigmoid output of Y (1, T, n_mels)."""
    return rn.SSRN(P, np.asarray(Y, np.float64))[1]


def windowed_ssrn64(P, Y, length, chunk, left, right, r=4):
    """Float64 SSRN of Y (T, n_mels) on the grid: the committed rows of every window, concatenated (r length, F)."""
    rows = []
    for a, e, s, t, _ in chunks(length, chunk, left, right):
        Z = ssrn64(P, Y[None, s:t])[0]
        rows.append(Z[r * (a - s):r * (e - s)])
    return np.concatenate(rows)
