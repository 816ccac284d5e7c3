"""Long-form synthesis on the GPU (dc_tts_b200/longform.py, csrc/kernels_longform.cu, SSRN past max_T):
  - Engine.join_rows against the numpy restatement of the join, bit for bit, zeros past each text's rows;
  - synthesize_texts against the same chain run by hand (decode, numpy join, ragged SSRN, ragged Griffin-Lim), bit for bit;
  - SSRN at 2 and 5 max_T: each utterance of a ragged call equals its own call (wgmma), and every block is within tau S of
    its float64 reference (tests/ref_forward_blocks.py) on both kernel sets; T <= max_T calls keep their bits and launches
    after the workspace grew;
  - the vocoder at 4000+ magnitude frames against the float32 oracle, and ragged against single calls;
  - the refusals: a workspace that cannot be allocated, bad pause and piece arguments.
Random weights never reach a piece's EOS: the stop positions come from a full run's window history, as
tools/bench_until_eos.py takes them, so that the pieces have lengths in proportion to their texts."""
import json
import os

import numpy as np
import pytest
import torch

import ref_forward_blocks as rf
from ref_longform import join_rows_reference
from dc_tts_b200 import longform as lf
from dc_tts_b200.arch import NETWORKS
from dc_tts_b200.data_load import utterance_lengths
from dc_tts_b200.engine import DcttsError, Engine
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params
from dc_tts_b200.utils import spectrograms2wavs
from oracle import ref_vocoder as rv

pytestmark = pytest.mark.gpu

TP = pytest.mark.parametrize("tp", [1, 0], ids=["tc", "fp32"])
TAU = {1: rf.TAU_TC, 0: rf.TAU_FP32}
BYTES_PER_FRAME = 98688          # r (scratch 2048 + 2 x 1028 floats + 4 x 1032 halfs) at c 512, d 256, F 1025

TEXTS = [
    ("It was the best of times, it was the worst of times, it was the age of wisdom, it was the age of foolishness, it "
     "was the epoch of belief, it was the epoch of incredulity. It was the season of Light, it was the season of "
     "Darkness! Was it the spring of hope, or the winter of despair?"),
    "Short one.",
    ("We had everything before us, we had nothing before us; we were all going direct to Heaven, we were all going "
     "direct the other way. In short, the period was so far like the present period, that some of its noisiest "
     "authorities insisted on its being received, for good or for evil, in the superlative degree of comparison only."),
]


@pytest.fixture
def eng(engine):
    yield engine
    engine.set_tensor_path(1)
    engine.set_option("chain_history", 0)


def realistic_stop_pos(e, L):
    """Per piece, the stop position whose until-EOS length is nearest to (its characters) x max_T / max_N."""
    _, Pf, _, _ = e.text2mel_generate(L)
    m = Pf.cpu().numpy()[:, 1:]
    chars = (np.asarray(L) > 0).sum(1)
    target = np.maximum(np.round(chars * hp.max_T / hp.max_N), 2)
    sp = np.zeros(len(L), np.int64)
    for b in range(len(L)):
        first = [0] + [j for j in range(1, m.shape[1]) if m[b, j] > m[b, j - 1]]
        j = min(first, key=lambda f: abs(f + 1 - target[b]))
        sp[b] = 0 if j == 0 else int(m[b, j])
    return sp, utterance_lengths(m, sp, 0, steps=hp.max_T)


# ---------------------------------------------------------------------------------------------- the join
JOIN_CASES = {
    "ragged": ([0, 0, 0, 1, 2, 2], [8, 4, 0, 0, 8, 0]),
    "zero pause": ([0, 0, 1, 1, 1], [0, 0, 0, 0, 0]),
    "one piece": ([0], [0]),
    "K=1": ([0, 0, 0, 0, 0, 0, 0], [8, 4, 4, 8, 0, 8, 0]),
    "many pieces": ([0] * 37 + [1] * 2, [4 if i % 3 else 8 for i in range(36)] + [0, 8, 0]),
}


@pytest.mark.parametrize("case", list(JOIN_CASES))
def test_join_rows_equals_numpy(eng, case):
    text, pause = JOIN_CASES[case]
    P, K, T = len(text), max(text) + 1, hp.max_T
    rng = np.random.default_rng(len(case))
    Y = rng.uniform(0, 1, (P, T, hp.n_mels)).astype(np.float32)
    n = rng.integers(1, T + 1, P).astype(np.int32)
    n[0], n[-1] = T, 1 if P > 1 else T
    for silence in (1e-8, 0.25):
        out, m = eng.join_rows(torch.from_numpy(Y), torch.from_numpy(n), text, pause, K, silence)
        T_out = out.shape[1]
        assert T_out == max(np.bincount(text, weights=T + np.array(pause), minlength=K))
        ref, mr = join_rows_reference(Y, n, text, pause, K, silence, T_out)
        assert np.array_equal(m.cpu().numpy(), mr)
        assert np.array_equal(out.cpu().numpy(), ref), case       # includes the zeros past each text's rows


def test_join_rows_clamps_device_lengths(eng):
    """Lengths outside [0, T] from the device are clamped, as ragged SSRN clamps them: no row outside a piece is read."""
    T = 16
    Y = torch.rand(3, T, hp.n_mels)
    n = np.array([-5, T + 9, 7], np.int32)
    out, m = eng.join_rows(Y, torch.from_numpy(n), [0, 0, 0], [2, 3, 0], 1)
    ref, mr = join_rows_reference(Y.numpy(), n, [0, 0, 0], [2, 3, 0], 1, 1e-8, out.shape[1])
    assert np.array_equal(m.cpu().numpy(), mr) and mr[0] == 2 + T + 3 + 7
    assert np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("text,pause,match", [
    ([0, 0, 1], [8, -1, 0], "pause of -1"),
    ([0, 0, 1], [8, 4, 0], "0 after a text's last piece"),
    ([0, 0, 1], [8, 0, 3], "0 after a text's last piece"),
    ([0, 1, 0], [0, 0, 0], "must follow the previous text's"),
    ([0, 2, 2], [0, 0, 0], "at least one piece"),
    ([1, 1, 2], [0, 0, 0], "at least one piece"),
])
def test_join_rows_refuses_bad_pieces(eng, text, pause, match):
    Y = torch.rand(3, 8, hp.n_mels)
    before = eng.launch_count()
    with pytest.raises(DcttsError, match=match):
        eng.join_rows(Y, torch.full((3,), 4, dtype=torch.int32), text, pause, 3)
    assert eng.launch_count() == before


def test_join_rows_refuses_bad_shapes(eng):
    with pytest.raises(DcttsError, match="P lengths"):
        eng.join_rows(torch.rand(2, 8, hp.n_mels), torch.ones(3, dtype=torch.int32), [0, 0], [0, 0], 1)
    with pytest.raises(DcttsError, match=r"\[0, K = 1\)"):
        eng.join_rows(torch.rand(2, 8, hp.n_mels), torch.ones(2, dtype=torch.int32), [0, 1], [0, 0], 1)
    with pytest.raises(ValueError, match="pause"):
        lf.synthesize_texts(eng, ["a"], pause=(8, -4))


# ---------------------------------------------------------------------------------------------- the whole chain
@TP
def test_synthesize_texts_equals_the_chain_by_hand(eng, tp):
    eng.set_tensor_path(tp)
    pieces, owner, pauses = lf.plan(TEXTS)
    L = lf.encode_pieces(pieces)
    sp, n_expect = realistic_stop_pos(eng, L)
    wavs, report = lf.synthesize_texts(eng, TEXTS, stop_pos=sp, momentum=0.5)
    # by hand: the decode, the numpy join, ragged SSRN, ragged Griffin-Lim
    Y, _, n = eng.text2mel_generate_until(L, stop_pos=sp)
    n_host = n.cpu().numpy()
    assert np.array_equal(n_host, n_expect)
    M, m = join_rows_reference(Y.cpu().numpy(), n_host, owner, pauses, len(TEXTS))
    assert m.max() > hp.max_T                                 # the longest text runs SSRN past max_T
    _, Z = eng.ssrn(torch.from_numpy(M), want_logits=False, lengths=torch.from_numpy(m))
    ref = spectrograms2wavs(Z, lengths=hp.r * m, momentum=0.5, engine=eng)
    assert len(wavs) == len(TEXTS)
    for k in range(len(TEXTS)):
        assert np.array_equal(wavs[k], ref[k]), k
        assert report[k]["frames"] == m[k]
    flat = [p for r in report for p in r["pieces"]]
    assert [p["text"] for p in flat] == [s for s, _ in pieces] and [p["pause"] for p in flat] == [k for _, k in pieces]
    assert [p["frames"] for p in flat] == n_host.tolist()
    assert all(p["eos"] for p in flat)


def test_synthesize_texts_reports_pieces_that_miss_their_eos(eng):
    """With the default stop positions (each piece's EOS) the random weights do not get through a 170-character piece in
    max_T frames: every piece runs max_T frames and the report says so."""
    sentence = " ".join(["word"] * 34) + "."
    wavs, report = lf.synthesize_texts(eng, [sentence + " " + sentence])
    assert [(p["frames"], p["eos"]) for p in report[0]["pieces"]] == [(hp.max_T, False), (hp.max_T, False)]
    assert report[0]["frames"] == 2 * hp.max_T + 8 and len(wavs) == 1


def test_long_form_synthesize_and_cli(tmp_path, monkeypatch):
    """synthesize(long_form=True) writes one wav per line of the sentences file, and the CLI one per line of its input,
    each that line's synthesize_texts."""
    from scipy.io.wavfile import read as read_wav

    from dc_tts_b200 import engine as engine_mod
    from dc_tts_b200.synthesize import synthesize
    lines = ["Glue the sheet. To the dark blue background, with care!", "It is easy."]
    sent = tmp_path / "sentences.txt"
    sent.write_text("header\n" + "".join("%d. %s\n" % (i + 1, t) for i, t in enumerate(lines)))
    monkeypatch.setattr(hp, "sampledir", str(tmp_path / "samples"))
    e = Engine(0)
    prev = engine_mod._default
    engine_mod.set_engine(e)
    try:
        wavs, report = synthesize(params=init_params(0), sentences=str(sent), long_form=True)
        ref, _ = lf.synthesize_texts(e, lines)
        for i in range(len(lines)):
            sr, w = read_wav(str(tmp_path / "samples" / ("%d.wav" % (i + 1))))
            assert sr == hp.sr and np.array_equal(w, ref[i]) and np.array_equal(wavs[i], ref[i])
        assert not os.path.exists(tmp_path / "samples" / "3.wav")
        infile = tmp_path / "in.txt"
        infile.write_text(lines[1] + "\n\n" + lines[0] + "\n")
        lf.main([str(infile), str(tmp_path / "out")])
        for i, j in ((1, 1), (2, 0)):
            assert np.array_equal(read_wav(str(tmp_path / "out" / ("%d.wav" % i)))[1], ref[j])
        rep = json.loads((tmp_path / "out" / "report.json").read_text())
        assert [r["frames"] for r in rep] == [report[1]["frames"], report[0]["frames"]]
    finally:
        engine_mod.set_engine(prev)
        e.close()


# ---------------------------------------------------------------------------------------------- SSRN past max_T
def _mels(B, T, seed):
    return torch.from_numpy(np.random.default_rng(seed).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32))


def _long_lengths(B, T):
    n = [T, T - 1, 2 * hp.max_T + 1, 640, 1, 129, hp.max_T, T // 2 + 3][:B]
    return [min(k, T) for k in n]


@TP
@pytest.mark.parametrize("mult", [2, 5])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_ssrn_ragged_past_max_t_equals_each_utterance_alone(eng, tp, mult, B):
    eng.set_tensor_path(tp)
    T = mult * hp.max_T
    n = _long_lengths(B, T)
    Y = _mels(B, T, 100 * mult + B).to(eng.device)
    Yr = Y.clone()
    for b, k in enumerate(n):
        Yr[b, k:] = float("nan")
    Z = torch.full((B, hp.r * T, eng.F), -7.0, device=eng.device)
    lg, Z = eng.ssrn(Yr, out=Z, lengths=torch.tensor(n, dtype=torch.int32, device=eng.device))
    lg, Z = lg.cpu(), Z.cpu()
    for b, k in enumerate(n):
        lg1, Z1 = eng.ssrn(Y[b:b + 1, :k])
        assert torch.equal(Z[b, :hp.r * k], Z1[0].cpu()) and torch.equal(lg[b, :hp.r * k], lg1[0].cpu()), (tp, b, k)
        assert not Z[b, hp.r * k:].any() and not lg[b, hp.r * k:].any(), (tp, b, k)


def _edge_rows(n):
    rows = {0, 1, 2, n - 2, n - 1}
    for e in range(128, n, 128):
        rows.update((e - 1, e))
    return np.array(sorted(r for r in rows if 0 <= r < n))


def _check_blocks(e, P, tp, n):
    """Every SSRN block of the last call on the tile-edge rows of each utterance's live rows, against its float64
    reference from the block's own input rows; rows past each utterance's live rows exactly 0."""
    layers = NETWORKS["SSRN"]()
    prm = [rf.block_params(P, "SSRN", l) for l in layers]
    x = e.chain_history("ssrn", 0, "input")[0].cpu().numpy()
    worst = 0.0
    for i, l in enumerate(layers):
        out, joined = e.chain_history("ssrn", i, "output")
        out = out.cpu().numpy()
        for b, k in enumerate(n):
            ins, live = rf.live_rows(layers, k)
            rows = _edge_rows(live[i])
            ref, S = rf.block_rows(prm[i], l, x[b, :ins[i]], rows)
            if joined:
                S = S + rf.S_PLANES
            err = np.abs(out[b, rows].astype(np.float64) - ref)
            r = np.where(S > 0, err / np.where(S > 0, S, 1), np.where(err > 0, np.inf, 0.0))
            worst = max(worst, float(r.max()))
            assert r.max() <= TAU[tp], (tp, l.scope, b, k, float(r.max()))
            assert not out[b, live[i]:].any(), (tp, l.scope, b, k)
        x = out
    return worst


@TP
@pytest.mark.parametrize("mult", [2, 5])
def test_ssrn_past_max_t_blocks_vs_float64(eng, params, tp, mult):
    eng.set_tensor_path(tp)
    eng.set_option("chain_history", 1)
    T = mult * hp.max_T
    Y = _mels(1, T, 7 * mult)
    eng.ssrn(Y)
    worst = _check_blocks(eng, params, tp, [T])
    if tp == 1:                       # ragged at the long length (the fp32 kernels run a ragged chain per utterance)
        n = _long_lengths(3, T)
        Y = _mels(3, T, 8 * mult)
        eng.ssrn(Y, lengths=np.array(n))
        worst = max(worst, _check_blocks(eng, params, tp, n))
    print("SSRN at T = %d, tp %d: worst err / S %.3g (tau %.3g)" % (T, tp, worst, TAU[tp]))


@TP
def test_short_calls_keep_their_bits_and_launches_after_a_grow(params, tp):
    e = Engine(0)
    try:
        e.load_params(params)
        e.set_tensor_path(tp)
        Y = _mels(4, hp.max_T, 3).to(e.device)
        n = torch.tensor([hp.max_T, 1, 100, 129], dtype=torch.int32, device=e.device)

        def run():
            l0 = e.launch_count()
            a = e.ssrn(Y)
            l1 = e.launch_count()
            b = e.ssrn(Y, lengths=n)
            l2 = e.launch_count()
            return [t.cpu() for t in a + b], (l1 - l0, l2 - l1)

        before, launches = run()
        bytes0 = e.reserve_frames(4, hp.max_T)
        grown = e.reserve_frames(8, 5 * hp.max_T)
        assert grown == 8 * 5 * hp.max_T * BYTES_PER_FRAME and grown > bytes0
        assert e.reserve_frames(2, hp.max_T) == grown              # never shrinks
        e.ssrn(_mels(8, 5 * hp.max_T, 4), want_logits=False)
        after, launches_after = run()
        assert launches_after == launches
        for x, y in zip(before, after):
            assert torch.equal(x, y)
    finally:
        e.close()


def test_workspace_that_cannot_be_allocated_is_refused(eng):
    Y = _mels(2, 50, 5).to(eng.device)
    ref = eng.ssrn(Y)[1].cpu()
    want = (1 << 20) * BYTES_PER_FRAME
    with pytest.raises(DcttsError, match=r"1 utterances of 1048576 frames need a synthesis workspace of %d bytes "
                                         r"\(98688 bytes per frame\), which cannot be allocated" % want):
        eng.reserve_frames(1, 1 << 20)
    with pytest.raises(DcttsError, match="more than 2\\^31 - 1"):
        eng.reserve_frames(1 << 10, 1 << 20)
    with pytest.raises(DcttsError, match="need B >= 1 and T >= 1"):
        eng.reserve_frames(0, 10)
    assert torch.equal(eng.ssrn(Y)[1].cpu(), ref)                  # the handle is as it was


# ---------------------------------------------------------------------------------------------- the vocoder at length
def test_vocoder_at_paragraph_length(eng):
    """4200 magnitude frames (5 max_T reduced frames): the de-emphasis carry over ~1.15 M samples, the trim energies and
    the window sum-square table at that length, against the float32 oracle to 2e-3 of the peak as the other vocoder tests
    hold it; the ragged call equals the single calls bit for bit."""
    T, n_iter = hp.r * 5 * hp.max_T, 3
    mag = np.random.default_rng(42).uniform(0.1, 0.95, (2, T, eng.F)).astype(np.float32)
    mag[1, T // 3:] *= 0.05
    mag[1, 2 * T // 3:] = 0.0
    n = [T, 4001]
    wav, trim = eng.spectrogram2wav(mag, n_iter=n_iter, lengths=n)
    wav = wav.cpu().numpy()
    for b, k in enumerate(n):
        w1, t1 = eng.spectrogram2wav(mag[b:b + 1, :k], n_iter=n_iter)
        Ly = hp.hop_length * (k - 1)
        assert np.array_equal(wav[b, :Ly], w1[0].cpu().numpy()) and not wav[b, Ly:].any()
        assert np.array_equal(trim[b], t1[0])
        _, se, full = rv.spectrogram2wav(mag[b, :k], n_iter=n_iter)
        scale = np.abs(full).max()
        assert np.abs(wav[b, :Ly] - full).max() < 2e-3 * scale, (b, np.abs(wav[b, :Ly] - full).max(), scale)
        assert abs(int(trim[b, 0]) - se[0]) <= 512 and abs(int(trim[b, 1]) - se[1]) <= 512
