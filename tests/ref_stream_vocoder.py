"""ORACLE (test infrastructure) -- the streaming Griffin-Lim vocoder (dctts_vocoder_stream_*, DESIGN.md section 8i)
restated in float64 for one utterance, on the stage references of tests/ref_vocoder_stages.py.

A push appends amplitude frames; with A frames received, one step is Griffin-Lim on the prefix [0, A) (a signal of
Ly = hop (A - 1) samples, reflect-padded at both of its ends as librosa.stft pads it) with the samples below the committed
count c held at their committed values:
  * active frames [f_lo, A): f_lo is the first frame whose window reaches past sample c; the frames below it touch no
    sample >= c, so they keep their X and take no part;
  * new frames [A_prev, A) start at X = S (zero phase), E = 0; the other active frames keep X and E (warm start);
  * each of n_iter iterations: istft of the active frames into samples [c, Ly), stft of the active frames, phase update
    (fast Griffin-Lim with momentum, as tests/ref_fast_griffin_lim.py); then one more istft;
  * commit: everything (Ly) on the final push, else up to the support start of frame t_r - MARGIN, t_r the first frame
    whose window reaches the reflected tail (sample >= Ly);
  * the committed samples [c, c') are de-emphasised (scipy.signal.lfilter) from the carried float64 state.
"""
import numpy as np
import scipy.signal

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_vocoder as rv

# The library's look-ahead margin in frames (api_audio.cu: VOC_STREAM_MARGIN)
MARGIN = 0


def window_bounds(n_fft, win):
    """(a0, a1): frame t's window covers the samples [hop t + a0, hop t + a1) of the centre-trimmed signal."""
    lpad = (n_fft - win) // 2
    return lpad - n_fft // 2, lpad + win - n_fft // 2


def first_active_frame(c, n_fft, hop, win):
    """The first frame whose window reaches a sample >= c."""
    _, a1 = window_bounds(n_fft, win)
    return 0 if c < a1 else (c - a1) // hop + 1


def commit_end(c, A, final, n_fft, hop, win, margin=MARGIN):
    """The committed sample count after a step on A frames that starts from c."""
    Ly = hop * (A - 1)
    if final:
        return Ly
    a0, a1 = window_bounds(n_fft, win)
    t_r = max(0, -(-(Ly - a1 + 1) // hop))          # first frame reading a sample >= Ly (the reflected tail)
    return min(Ly, max(c, hop * (t_r - margin) + a0))


class StreamVocoder:
    """One utterance.  push(S_rows (k, F) float64 amplitude, final) -> the newly committed de-emphasised samples
    (float64).  y holds the Griffin-Lim waveform before de-emphasis; spans lists each push's [c, c')."""

    def __init__(self, n_fft, hop, win, n_iter, momentum=0.0, margin=MARGIN, preemphasis=None):
        self.n_fft, self.hop, self.win, self.n_iter, self.margin = n_fft, hop, win, n_iter, margin
        self.alpha = momentum / (1.0 + momentum)
        self.pre = hp.preemphasis if preemphasis is None else preemphasis
        self.w = rv.hann_padded(n_fft, win, np.float64)
        F = 1 + n_fft // 2
        self.S = np.zeros((0, F))
        self.X = np.zeros((0, F), np.complex128)
        self.E = np.zeros((0, F), np.complex128)
        self.y = np.zeros(0)
        self.c = 0
        self.state = 0.0
        self.ended = False
        self.spans = []

    def _istft(self, lo, A):
        """Samples [c, Ly) of librosa.istft of the A-frame spectrum (frames below lo add nothing there)."""
        n_fft, hop = self.n_fft, self.hop
        Xs = self.X[lo:A].copy()
        Xs[:, 0] = Xs[:, 0].real
        Xs[:, -1] = Xs[:, -1].real
        fr = np.fft.irfft(Xs, n=n_fft, axis=-1) * self.w
        n = n_fft + hop * (A - 1)
        y = np.zeros(n)
        for i, t in enumerate(range(lo, A)):
            y[t * hop:t * hop + n_fft] += fr[i]
        wss = rv.window_sumsquare(A, n_fft, hop, self.win, np.float64)
        nz = wss > np.finfo(np.float64).tiny
        y[nz] /= wss[nz]
        return y[n_fft // 2 + self.c:n - n_fft // 2]

    def _stft(self, lo, A):
        n_fft, hop = self.n_fft, self.hop
        yp = np.pad(self.y[:hop * (A - 1)], n_fft // 2, mode="reflect")
        idx = np.arange(n_fft)[None, :] + hop * np.arange(lo, A)[:, None]
        return np.fft.rfft(yp[idx] * self.w, axis=-1)

    def push(self, S_rows, final=False):
        assert not self.ended, "push after final"
        A_prev = self.S.shape[0]
        S_rows = np.asarray(S_rows, np.float64)
        self.S = np.concatenate([self.S, S_rows])
        self.X = np.concatenate([self.X, S_rows.astype(np.complex128)])
        self.E = np.concatenate([self.E, np.zeros_like(S_rows, np.complex128)])
        A = self.S.shape[0]
        self.ended = bool(final)
        if A < 2:
            assert not final, "an utterance needs at least 2 frames"
            return np.zeros(0)
        Ly = self.hop * (A - 1)
        if self.y.shape[0] < Ly:
            self.y = np.concatenate([self.y, np.zeros(Ly - self.y.shape[0])])
        lo = first_active_frame(self.c, self.n_fft, self.hop, self.win)
        for _ in range(self.n_iter):
            self.y[self.c:Ly] = self._istft(lo, A)
            est = self._stft(lo, A)
            cc = est - self.alpha * self.E[lo:A] if self.alpha != 0 else est
            self.E[lo:A] = est
            self.X[lo:A] = self.S[lo:A] * (cc / np.maximum(1e-8, np.abs(cc)))
        self.y[self.c:Ly] = self._istft(lo, A)
        c_new = commit_end(self.c, A, final, self.n_fft, self.hop, self.win, self.margin)
        seg = self.y[self.c:c_new]
        out = np.zeros(0)
        if seg.size:
            out, zf = scipy.signal.lfilter([1], [1, -self.pre], seg, zi=[self.pre * self.state])
            self.state = float(out[-1])
        self.spans.append((self.c, c_new))
        self.c = c_new
        return out


def stream(S, chunk, n_fft, hop, win, n_iter, momentum=0.0, margin=MARGIN):
    """The whole (T, F) amplitude S pushed `chunk` frames at a time, the last push final -> (list of committed sample
    arrays, the StreamVocoder)."""
    v = StreamVocoder(n_fft, hop, win, n_iter, momentum, margin)
    T = S.shape[0]
    outs = []
    for a in range(0, T, chunk):
        outs.append(v.push(S[a:a + chunk], final=a + chunk >= T))
    return outs, v
