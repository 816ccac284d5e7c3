"""Parity against the REFERENCE'S OWN SOURCE.  tests/golden/refshim_*.npz were produced by importing
/root/reference/{modules,networks,train}.py and executing Graph(mode="synthesize") under the TensorFlow API
stand-in tests/golden/tf_shim.py (generator: tests/golden/make_golden_refshim.py).  They pin everything the
reference's Python decides (topology, dilations, paddings, scopes/variable names, the decoder shift, the window
mask); the TF op semantics themselves are the shim's restatement (see its header).

  * CPU: the oracle's two restatements vs these fixtures, and vs refshim_live.npz / refshim_host.npz (a few decode
    steps, the variable names the graph asks for, the text adaptor, the training constants, the vocoder and feature
    composition; generator: tests/golden/make_golden_refchecks.py).  Where a checkout of the reference is present the
    same checks also run against the reference code live.
  * GPU: the CUDA path vs these fixtures."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, golden
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text
from oracle import ref_numpy as rn
from oracle import ref_torch as rt

TOL = 1e-3            # north_star: max-abs on mel / linear magnitudes
HAVE_REF = os.path.isfile("/root/reference/networks.py")


@pytest.fixture(scope="module")
def P():
    return init_params(0, "perturbed")


def _inputs_forward():
    L = synthetic_text(1, 60, seed=3)
    mels = np.random.default_rng(11).uniform(0, 1, (1, hp.max_T, hp.n_mels)).astype(np.float32)
    return L, mels, np.array([7], np.int32)


def test_oracle_full_graph_vs_reference_code(P):
    g = golden("refshim_t2m_forward.npz")
    L, mels, pma = _inputs_forward()
    o = rt.text2mel_forward(P, L, mels, pma)
    assert np.abs(o["Y"].numpy() - g["Y"]).max() < 2e-5
    assert np.array_equal(o["max_attentions"].numpy(), g["max_attentions"])
    assert np.abs(o["Q"].numpy()[:, ::10, :16] - g["Q_sub"]).max() < 1e-4
    assert np.abs(o["K"].numpy()[:, ::10, :16] - g["K_sub"]).max() < 1e-4
    assert np.abs(o["R"].numpy()[:, ::10, ::16] - g["R_sub"]).max() < 1e-4
    assert np.abs(o["alignments"].numpy()[:, 7:10, :] - g["align_win"]).max() < 1e-5
    # and the two fixture sets (oracle-made, reference-made) agree
    g0 = golden("t2m_forward.npz")
    assert np.abs(g0["Y"] - g["Y"]).max() < 2e-5 and np.array_equal(g0["max_attentions"], g["max_attentions"])


def test_oracle_ssrn_vs_reference_code(P):
    g = golden("refshim_ssrn_T12.npz")
    Y = np.random.default_rng(12).uniform(0, 1, (1, 12, hp.n_mels)).astype(np.float32)
    zl, z = rt.SSRN(P, torch.from_numpy(Y))
    assert np.abs(z.numpy() - g["Z"]).max() < 2e-5
    assert np.abs(zl.numpy()[:, :, ::8] - g["Z_logits_sub"]).max() < 5e-4
    zl2, z2 = rn.SSRN(P, Y)
    assert np.abs(np.asarray(z2) - g["Z"]).max() < 2e-5


def test_oracle_synthesis_loop_vs_reference_code():
    """210 free-running steps of the reference's loop (synthesize.py:45-57) on Harvard sentence 1: identical window
    trajectory, mel within float32 noise -- against the oracle-made fixture of the same run."""
    g, g0 = golden("refshim_synth_harvard1.npz"), golden("synth_harvard1.npz")
    assert np.array_equal(g["L"], g0["L"])
    assert np.array_equal(g["p_hist"], g0["p_hist"])
    assert np.abs(g["Y"] - g0["Y"]).max() < 1e-4
    assert np.abs(g["Z_sub"] - g0["Z_sub"]).max() < 1e-4


def test_oracle_few_steps_vs_reference_output(P):
    """A few steps of the reference's loop and its SSRN on their first 8 frames, and the variables its graph asked for."""
    g = golden("refshim_live.npz")
    L = synthetic_text(2, 40, seed=5)
    with torch.no_grad():
        o = rt.synthesize(P, L, steps=3, literal=True, record=True)
    assert np.abs(g["Y3"] - o["Y"].numpy()[:, :3]).max() < 2e-5
    assert np.array_equal(g["p_hist"], o["p_hist"].numpy()[:, :3])
    _, z2 = rt.SSRN(P, torch.from_numpy(g["Y8"].copy()))
    assert np.abs(g["Z8"] - z2.numpy()).max() < 2e-5
    # the graph asked for exactly the variables of the schema (SURVEY.md App. C)
    assert set(g["requested"].tolist()) == set(P)


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_reference_code_live_few_steps(P):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tf_shim
    store = tf_shim.Store(P)
    tf_shim.install(store)
    L = synthetic_text(2, 40, seed=5)
    r = tf_shim.synthesize(L, steps=3, with_ssrn=False)
    with torch.no_grad():
        o = rt.synthesize(P, L, steps=3, literal=True, record=True)
    assert np.abs(r["Y"][:, :3] - o["Y"].numpy()[:, :3]).max() < 2e-5
    assert np.array_equal(r["p_hist"], o["p_hist"].numpy()[:, :3])
    _, z = tf_shim.run_ssrn(r["Y"][:, :8])
    _, z2 = rt.SSRN(P, torch.from_numpy(r["Y"][:, :8].copy()))
    assert np.abs(z - z2.numpy()).max() < 2e-5
    # the graph asked for exactly the variables of the schema (SURVEY.md App. C), with the schema's shapes
    assert store.requested == set(P)
    # an unknown or mis-shaped variable is an error, not a silent default
    bad = dict(P); bad["Text2Mel/TextEnc/C_2/conv1d/kernel"] = np.zeros((1, 128, 511), np.float32)
    tf_shim.install(tf_shim.Store(bad))
    with pytest.raises(ValueError):
        tf_shim.run_graph(L, np.zeros((2, hp.max_T, hp.n_mels), np.float32), np.zeros(2, np.int32))
    tf_shim.install(store)


# ------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_cuda_full_graph_vs_reference_code(engine, path):
    g = golden("refshim_t2m_forward.npz")
    L, mels, pma = _inputs_forward()
    Y, M, A = engine.text2mel_forward(L, mels, pma)
    assert np.abs(Y.cpu().numpy() - g["Y"]).max() < TOL
    assert np.array_equal(M.cpu().numpy(), g["max_attentions"])
    assert np.abs(A.cpu().numpy()[:, 7:10, :] - g["align_win"]).max() < 1e-4


@pytest.mark.gpu
def test_cuda_ssrn_vs_reference_code(engine, path):
    g = golden("refshim_ssrn_T12.npz")
    Y = np.random.default_rng(12).uniform(0, 1, (1, 12, hp.n_mels)).astype(np.float32)
    _, Z = engine.ssrn(Y, want_logits=False)
    assert np.abs(Z.cpu().numpy() - g["Z"]).max() < TOL


@pytest.mark.gpu
def test_cuda_synthesis_vs_reference_code(engine):
    """The CUDA-graph decode loop + SSRN vs the reference's own loop run under the shim (Harvard sentence 1)."""
    g = golden("refshim_synth_harvard1.npz")
    Y, Pm, M, A = engine.text2mel_generate(g["L"], want_final_attention=True)
    assert np.array_equal(Pm.cpu().numpy(), g["p_hist"])
    assert np.abs(Y.cpu().numpy() - g["Y"]).max() < TOL
    assert np.array_equal(M.cpu().numpy(), g["max_attentions"])
    _, Z = engine.ssrn(Y, want_logits=False)
    assert np.abs(Z.cpu().numpy()[:, ::8, ::8] - g["Z_sub"]).max() < TOL


# ------------------------------------------------------------------------------------------- host-side pieces
def _vocoder_inputs():
    """(magnitudes, waveform): the seeded inputs of the vocoder / feature checks (make_golden_refchecks.py draws the same)."""
    rng = np.random.default_rng(0)
    mag = rng.uniform(0.2, 0.8, (40, 1 + hp.n_fft // 2)).astype(np.float32)
    t = np.arange(int(hp.sr * 0.8)) / hp.sr
    y = (0.2 * np.sin(2 * np.pi * 300 * t) + 0.02 * rng.standard_normal(t.size)).astype(np.float32)
    y[:2000] *= 1e-5
    return mag, y


def test_text_adaptor_vs_reference_output():
    """The reference's data_load.load_data("synthesize") ids on its harvard_sentences.txt and its vocabulary vs the mirror
    in dc_tts_b200/data_load.py: all 20 sentences, every id."""
    g = golden("refshim_host.npz")
    from dc_tts_b200.data_load import load_data, load_vocab
    mine = load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))
    assert g["ids"].shape == (20, hp.max_N) and g["ids"].dtype == np.int32
    assert np.array_equal(g["ids"], mine)
    char2idx, idx2char = load_vocab()
    vocab = g["vocab"].tolist()
    assert [idx2char[i] for i in range(len(idx2char))] == vocab and all(char2idx[c] == i for i, c in enumerate(vocab))
    assert np.array_equal(golden("refshim_synth_harvard1.npz")["L"], g["ids"][:1])


def test_training_constants_vs_reference_output():
    """utils.guided_attention (utils.py:134-140) and the Noam schedule (utils.py:141-145) as the reference computed them."""
    from oracle import ref_train as rtr
    g = golden("refshim_host.npz")
    np.testing.assert_allclose(g["guided_attention"], rtr.guided_attention(), rtol=0, atol=1e-7)
    for gs, v in zip(g["lr_steps"], g["lr"]):
        assert float(v) == pytest.approx(rtr.learning_rate(int(gs)), rel=1e-6)


def test_vocoder_and_feature_composition_vs_reference_output():
    """utils.spectrogram2wav (3 iterations) / load_spectrograms as the reference composed them (with the restated
    primitives standing in for librosa) vs the oracle's composition."""
    from oracle import ref_features as rf
    from oracle import ref_vocoder as rv
    g = golden("refshim_host.npz")
    mag, y = _vocoder_inputs()
    mine, _, _ = rv.spectrogram2wav(mag, n_iter=3)
    assert g["wav"].shape == mine.shape and np.abs(g["wav"] - mine).max() <= 1e-6 * max(1.0, np.abs(mine).max())
    mel2, mg2 = rf.load_spectrograms(y)
    assert g["mel"].shape == mel2.shape and g["mag"].shape == mg2.shape
    assert np.abs(g["mel"] - mel2).max() < 1e-6 and np.abs(g["mag"] - mg2).max() < 1e-6


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_text_adaptor_vs_reference_code(monkeypatch):
    """data_load.load_data("synthesize") of the reference itself (data_load.py:79-86) on its own harvard_sentences.txt
    vs the mirror in dc_tts_b200/data_load.py: all 20 sentences, every id."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tf_shim
    tf_shim.install(tf_shim.Store({}))
    import data_load as ref_dl
    import hyperparams as ref_hp
    monkeypatch.setattr(ref_hp.Hyperparams, "test_data", "/root/reference/harvard_sentences.txt")
    ref = ref_dl.load_data("synthesize")
    from dc_tts_b200.data_load import load_data, load_vocab
    mine = load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))
    assert ref.shape == (20, hp.max_N) and ref.dtype == np.int32
    assert np.array_equal(ref, mine)
    assert ref_dl.load_vocab() == load_vocab()
    assert np.array_equal(golden("refshim_synth_harvard1.npz")["L"], ref[:1])


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_training_constants_vs_reference_code():
    """utils.guided_attention (utils.py:134-140) and the Noam schedule (utils.py:141-145) of the reference itself."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tf_shim
    tf_shim.install(tf_shim.Store({}))
    import utils as ref_utils
    from oracle import ref_train as rtr
    np.testing.assert_allclose(ref_utils.guided_attention(), rtr.guided_attention(), rtol=0, atol=1e-7)
    for gs in (0, 1, 3999, 4000, 123456):
        assert float(ref_utils.learning_rate_decay(hp.lr, gs)) == pytest.approx(rtr.learning_rate(gs), rel=1e-6)


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_vocoder_and_feature_composition_vs_reference_code(monkeypatch):
    """utils.spectrogram2wav / get_spectrograms / load_spectrograms of the reference itself, with the absent `librosa`
    replaced by the restated primitives (oracle/ref_vocoder.py, ref_features.py): pins how the reference COMPOSES
    them (de-normalisation, power, Griffin-Lim loop, lfilter, trim; pre-emphasis, mel, dB, normalisation, reduction) --
    the primitives themselves stay a restatement."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import types
    import tf_shim
    tf_shim.install(tf_shim.Store({}))
    import utils as ref_utils
    from oracle import ref_features as rf
    from oracle import ref_vocoder as rv
    lib = types.SimpleNamespace(
        stft=lambda y, n_fft=None, hop_length=None, win_length=None: rv.stft(np.asarray(y, np.float32), n_fft, hop_length, win_length),
        istft=lambda S, hop_length=None, win_length=None, window="hann": rv.istft(S, hop_length, win_length),
        effects=types.SimpleNamespace(trim=lambda y: (lambda se: (y[se[0]:se[1]], se))(rv.trim_indices(np.asarray(y)))),
        filters=types.SimpleNamespace(mel=lambda sr, n_fft, n_mels: rf.mel_basis(sr, n_fft, n_mels)),
        load=lambda fpath, sr=None: (WAVS[fpath], sr))
    monkeypatch.setattr(ref_utils, "librosa", lib)
    import hyperparams as ref_hp
    monkeypatch.setattr(ref_hp.Hyperparams, "n_iter", 3)
    monkeypatch.setattr(hp, "n_iter", 3)
    rng = np.random.default_rng(0)
    mag = rng.uniform(0.2, 0.8, (40, 1 + hp.n_fft // 2)).astype(np.float32)
    ref_wav = ref_utils.spectrogram2wav(mag)
    mine, _, _ = rv.spectrogram2wav(mag, n_iter=3)
    assert ref_wav.shape == mine.shape and np.abs(ref_wav - mine).max() <= 1e-6 * max(1.0, np.abs(mine).max())
    t = np.arange(int(hp.sr * 0.8)) / hp.sr
    y = (0.2 * np.sin(2 * np.pi * 300 * t) + 0.02 * rng.standard_normal(t.size)).astype(np.float32)
    y[:2000] *= 1e-5
    WAVS = {"LJ001-0001.wav": y}
    fname, mel, mg = ref_utils.load_spectrograms("LJ001-0001.wav")
    mel2, mg2 = rf.load_spectrograms(y)
    assert fname == "LJ001-0001.wav" and mel.shape == mel2.shape and mg.shape == mg2.shape
    assert np.abs(mel - mel2).max() < 1e-6 and np.abs(mg - mg2).max() < 1e-6
