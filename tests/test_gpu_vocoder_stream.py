"""Streaming Griffin-Lim on the GPU (dctts_vocoder_stream_*, Engine.vocoder_stream).

  * One final push is dctts_spectrogram2wav_momentum with lengths, bit for bit (waveform and trims), at n_fft 1024, 2048
    and 4096, plain and with momentum.
  * Pushed in pieces, each push commits exactly the samples the float64 restatement (tests/ref_stream_vocoder.py)
    commits, and the waveform matches it within TAU of its norm, per utterance, at n_iter 0, 1 and 3.
  * Quality: streamed in 64-frame pieces with 50 iterations, 8 s signals reach a spectral convergence within 1.5x of
    whole-signal Griffin-Lim, plain and with momentum 0.99.
  * Refusals: rows after the final push, more frames than the stream holds, a final utterance of one frame, a close
    before every utterance is final; the handle stays usable.  Engine.close frees the streams still open on it.
Engines are built and run inside `at_rate`, because an engine reads hop and win from Hyperparams at call time.
"""
import numpy as np
import pytest

from dc_tts_b200.engine import DcttsError
from oracle import ref_features as rf
from oracle import ref_vocoder as rv
import ref_fast_griffin_lim as fg
import ref_stream_vocoder as sv
import ref_vocoder_stages as rs
from sample_rates import at_rate

pytestmark = pytest.mark.gpu
SR = {1024: 16000, 2048: 22050, 4096: 44100}
# norm-relative waveform error against float64, per (n_fft, n_iter), about 3x the worst measured on an H100 80GB HBM3 at
# 700 W (printed at the end of the module): n_iter 0: 3.01e-6, 2.37e-5, 2.61e-5; n_iter 1: 1.25e-5, 1.65e-4, 1.14e-4;
# n_iter 3 (momentum 0.99): 4.02e-3, 2.80e-4, 2.96e-4 at n_fft 1024, 2048, 4096.  Phase retrieval amplifies float32
# rounding in ill-conditioned bins from one iteration to the next, so the bound grows with n_iter.
TAU = {1024: (9e-6, 3.8e-5, 1.2e-2), 2048: (7.1e-5, 5e-4, 8.4e-4), 4096: (7.8e-5, 3.4e-4, 8.9e-4)}
_WORST = {}


@pytest.fixture(scope="module")
def engines():
    from dc_tts_b200.engine import Engine
    out = {}
    for n in SR:
        with at_rate(SR[n], n) as H:
            out[n] = Engine(0, hparams=H)
    yield out
    print("\nstreaming vocoder, worst |got - ref| / |ref|: " + ", ".join("%s %.3g" % (k, v) for k, v in sorted(_WORST.items())))
    for e in out.values():
        e.close()


def _stream(eng, mag, lengths, chunk, n_iter, momentum, T_cap=None):
    """Pushes mag (B, T, F) `chunk` rows per utterance at a time (utterance b has lengths[b] rows, final on its last
    piece) -> (per-utterance lists of the pushed pieces' samples, trims)."""
    B = mag.shape[0]
    vs = eng.vocoder_stream(B, T_cap or mag.shape[1] + 5, n_iter=n_iter, momentum=momentum)
    pieces = [[] for _ in range(B)]
    for a in range(0, max(lengths), chunk):
        counts = [max(0, min(chunk, L - a)) for L in lengths]
        final = [a < L <= a + chunk for L in lengths]
        out = vs.push(mag[:, a:a + chunk], counts, final)
        for b in range(B):
            if counts[b] or final[b]:
                pieces[b].append(out[b])
    return pieces, vs.close()


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("momentum", [0.0, 0.99])
def test_one_final_push_is_spectrogram2wav(engines, n, momentum):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        T, lengths = 60, [60, 2, 37]
        mag = rs.make_mag(np.random.default_rng(n), 3, T, n)
        wav, trim = eng.spectrogram2wav(mag, n_iter=5, lengths=lengths, momentum=momentum)
        pieces, trim_s = _stream(eng, mag, lengths, T, 5, momentum, T_cap=200)
        wav = wav.cpu().numpy()
        for b, L in enumerate(lengths):
            assert len(pieces[b]) == 1 and np.array_equal(pieces[b][0], wav[b, :H.hop_length * (L - 1)]), b
        assert np.array_equal(trim, trim_s)


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("n_iter", [0, 1, 3])
def test_pieces_match_the_float64_stream(engines, n, n_iter):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        hop, win = H.hop_length, H.win_length
        momentum = 0.99 if n_iter == 3 else 0.0
        mags = [rf.get_spectrograms(rs.signal(k, seconds=1.0, seed=n))[1] for k in rs.SIGNALS]
        lengths = [m.shape[0] - 7 * b for b, m in enumerate(mags)]
        T = max(lengths)
        mag = np.zeros((3, T, 1 + n // 2), np.float32)
        for b, L in enumerate(lengths):
            mag[b, :L] = mags[b][:L]
        chunk = 9
        pieces, _ = _stream(eng, mag, lengths, chunk, n_iter, momentum)
        for b, L in enumerate(lengths):
            S = rs.ref_prepare(mag[b, :L], H.power)
            ref, v = sv.stream(S, chunk, n, hop, win, n_iter, momentum)
            assert [p.size for p in pieces[b]] == [r.size for r in ref], b
            got, want = np.concatenate(pieces[b]).astype(np.float64), np.concatenate(ref)
            rel = float(np.linalg.norm(got - want) / np.linalg.norm(want))
            _WORST["n_fft %d n_iter %d" % (n, n_iter)] = max(_WORST.get("n_fft %d n_iter %d" % (n, n_iter), 0.0), rel)
            assert rel <= TAU[n][(0, 1, 3).index(n_iter)], (b, rel)


def _convergence(wav, S, n, hop, win, pre):
    """Spectral convergence of a de-emphasised waveform, pre-emphasis undone in float64."""
    x = wav.astype(np.float64)
    x[1:] = x[1:] - pre * wav[:-1].astype(np.float64)
    return fg.spectral_convergence(S, rv.stft(x, n, hop, win))


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("momentum", [0.0, 0.99])
def test_streamed_quality_is_within_the_bar(engines, n, momentum):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        mag = np.stack([rf.get_spectrograms(rs.signal(k, seconds=8))[1] for k in rs.SIGNALS])
        B, T, _ = mag.shape
        whole, _ = eng.spectrogram2wav(mag, n_iter=50, momentum=momentum)
        whole = whole.cpu().numpy()
        pieces, _ = _stream(eng, mag, [T] * B, 64, 50, momentum)
        for b, kind in enumerate(rs.SIGNALS):
            S = rs.amplitude(mag[b], H.power, np.float64)
            streamed = np.concatenate(pieces[b])
            sc_s = _convergence(streamed, S, n, H.hop_length, H.win_length, H.preemphasis)
            sc_w = _convergence(whole[b], S, n, H.hop_length, H.win_length, H.preemphasis)
            print("n_fft %d momentum %g %s: whole %.4f streamed %.4f (x%.3f)" % (n, momentum, kind, sc_w, sc_s, sc_s / sc_w))
            assert streamed.size == whole.shape[1]
            assert sc_s <= 1.5 * sc_w, (kind, sc_s, sc_w)


def test_refusals(engines):
    eng = engines[2048]
    with at_rate(SR[2048]):
        mag = np.full((2, 6, 1025), 0.5, np.float32)
        vs = eng.vocoder_stream(2, 10, n_iter=1)
        vs.push(mag, [6, 3], [True, False])
        with pytest.raises(DcttsError, match="utterance 0 has had its final push"):
            vs.push(mag, [1, 0], False)
        with pytest.raises(DcttsError, match="utterance 1 would have 13 frames, past T_cap = 10"):
            vs.push(np.full((2, 10, 1025), 0.5, np.float32), [0, 10])
        with pytest.raises(DcttsError, match="has not had its final push"):
            vs.close()
        vs = eng.vocoder_stream(1, 10, n_iter=1)
        with pytest.raises(DcttsError, match="utterance 0 ends with 1 frame"):
            vs.push(mag[:1], [1], True)
        vs.push(mag[:1], [2], True)
        assert vs.close().shape == (1, 2)
        wav, _ = eng.spectrogram2wav(mag, n_iter=1)             # the handle stays usable
        assert wav.shape == (2, 275 * 5)


def test_engine_close_frees_its_open_streams():
    """A stream left open is freed by Engine.close, before the handle it holds; using it afterwards is refused."""
    from dc_tts_b200.engine import Engine
    with at_rate(SR[2048]) as H:
        eng = Engine(0, hparams=H)
        vs = eng.vocoder_stream(1, 10, n_iter=1)
        vs.push(np.full((1, 3, 1025), 0.5, np.float32), [3])
        eng.close()
        with pytest.raises(DcttsError, match="the stream is closed"):
            vs.push(np.full((1, 1, 1025), 0.5, np.float32), [1])
        del vs
