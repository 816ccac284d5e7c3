"""Drop-in for the reference's synthesize.py (/root/reference/synthesize.py:21-64).

Same flow: load text -> build Graph(mode="synthesize") -> restore parameters -> mel
loop (:45-54) -> SSRN (:57) -> write one output per sentence.  Differences, all forced
by what exists offline: parameters are restored from the TF checkpoints under
hp.logdir-1 / hp.logdir-2 when they exist (dc_tts_b200/checkpoint.py reads the tensor
bundles without TensorFlow), else come from a name->array dict or the seeded initialiser.  The Griffin-Lim vocoder
(utils.py:67-114) runs on the GPU (dc_tts_b200/utils.py) and the wavs are written with
scipy.io.wavfile like the reference does.
"""
import os

import numpy as np

from .checkpoint import latest_checkpoint
from .data_load import load_data
from .engine import get_engine
from .hyperparams import Hyperparams as hp
from .params import init_params
from .train import Graph, Session


def _timing_of(g, L, wavs):
    """The attention-window path (B, T) and frame counts (B,) of each sentence of L spoken with the timing of its
    recording (one WAV file per sentence, at any sample rate)."""
    from .utils import load_spectrograms_batch
    if len(wavs) != len(L):
        raise ValueError("timing_from: %d recordings for %d sentences" % (len(wavs), len(L)))
    _, mels, _, t = load_spectrograms_batch(list(wavs), g.engine, resample=True)
    over = np.flatnonzero(t > hp.max_T)
    if over.size:
        raise ValueError("timing_from: %s has %d frames, more than max_T = %d" % (wavs[over[0]], t[over[0]], hp.max_T))
    path, _, _, _ = g.align(L, mels, t)
    return path, t


def _restore(engine, params, seed, allow_random_init):
    """synthesize.py:31-41: the caller's dictionary, else the parameters already on the engine, else the checkpoints."""
    if params is not None:
        engine.load_params(params)
        print("Parameters loaded from the caller's dictionary")
    elif engine.params_loaded:
        print("Using the parameters already committed to the engine")
    else:
        ck1, ck2 = latest_checkpoint(hp.logdir + "-1"), latest_checkpoint(hp.logdir + "-2")
        if ck1 and ck2:
            engine.restore(hp.logdir + "-1", hp.logdir + "-2")
            print("Text2Mel Restored!")
            print("SSRN Restored!")
        elif allow_random_init:
            engine.load_params(init_params(seed))
            print("WARNING: no checkpoint -- seeded random weights (allow_random_init=True); the output is noise")
        else:
            missing = [d for d, c in ((hp.logdir + "-1", ck1), (hp.logdir + "-2", ck2)) if not c]
            raise FileNotFoundError("no checkpoint under %s (reference: Saver.restore(sess, None) fails); pass params=..., "
                                    "or allow_random_init=True for seeded random weights" % " and ".join(missing))


def _synthesize_long_form(params, sentences, write, seed, allow_random_init, tail, momentum):
    from .longform import read_texts, synthesize_texts
    texts = read_texts(sentences or hp.test_data, header=True)
    g = Graph(mode="synthesize")
    with Session():
        _restore(g.engine, params, seed, allow_random_init)
        wavs, report = synthesize_texts(g.engine, texts, tail=tail, momentum=momentum)
    if write:
        from scipy.io.wavfile import write as write_wav
        if not os.path.exists(hp.sampledir):
            os.makedirs(hp.sampledir)
        for i, wav in enumerate(wavs):
            print("Working on file", i + 1)
            write_wav(os.path.join(hp.sampledir, "{}.wav".format(i + 1)), hp.sr, wav)
    return wavs, report


def synthesize(params=None, sentences=None, fast=True, write=True, seed=0, vocoder=True, allow_random_init=False,
               until_eos=False, tail=0, momentum=0.0, duration_scale=1.0, timing_from=None, long_form=False):
    """`params`: a name -> array dict to use instead of the checkpoints.  Without it the latest checkpoints of
    hp.logdir-1 (Text2Mel) and hp.logdir-2 (SSRN) are restored, and a missing one RAISES like the reference's
    `saver.restore(sess, None)` does (synthesize.py:33,39) -- seeded random weights are used only when the caller asks
    for them (`allow_random_init=True`, benchmarks and smoke tests) or has already loaded parameters into the engine.

    `until_eos=True`: each utterance ends `tail` frames after its attention reaches the EOS of its text
    (Graph.generate_until_eos).  SSRN and the vocoder then run once each over the batch at its longest length, with a
    length per utterance: each wav is Griffin-Lim of that utterance's r * length magnitude frames.  Y and Z rows past each
    length are 0.

    `momentum`: the vocoder's fast Griffin-Lim update (librosa's griffinlim(momentum=...)); 0 is the reference's plain
    Griffin-Lim.

    `duration_scale`: speaking rate, > 1 slower.  At any value other than 1.0 each utterance is first decoded to its EOS
    as with `until_eos=True`, its attention-window history is stretched by that factor (utils.stretch_path), and the
    utterance is decoded again along the stretched path (Graph.generate_along); SSRN and the vocoder then run with the
    stretched lengths.  1.0 leaves every other route exactly as it is.

    `timing_from`: a list of WAV files, one recording per sentence.  Each sentence is spoken with the timing of its
    recording: the recording's features (resampled to hp.sr when needed) are aligned to the sentence (Graph.align), the
    recovered path is stretched by `duration_scale` when that is not 1, and the sentence is decoded along it
    (Graph.generate_along); SSRN and the vocoder run with each recording's frame count (or the stretched one).  A
    recording longer than max_T frames is refused.  None leaves every other route exactly as it is.

    `long_form=True`: each line of the sentences file (the first line a header, a leading "N. " removed, as load_data
    reads it) is one text of any length, read by longform.synthesize_texts (split into pieces, decoded to their ends as
    one batch, joined on the device, SSRN and Griffin-Lim once per text), with `tail` and `momentum`; one wav per line.
    Returns (wavs, report).  False leaves every other route exactly as it is."""
    if long_form:
        return _synthesize_long_form(params, sentences, write, seed, allow_random_init, tail, momentum)
    # Load data
    L = load_data("synthesize", sentences)

    # Load graph
    g = Graph(mode="synthesize")
    print("Graph loaded")

    with Session() as sess:
        # Restore parameters (synthesize.py:31-41)
        _restore(g.engine, params, seed, allow_random_init)

        lengths = None
        if timing_from is not None or until_eos or duration_scale != 1.0:
            if timing_from is not None:
                P, n = _timing_of(g, L, timing_from)
            else:
                Y, P, n = g.generate_until_eos(L, tail=tail)
            if duration_scale != 1.0:
                from .utils import stretch_path
                P, n = stretch_path(P, n, duration_scale)
            if timing_from is not None or duration_scale != 1.0:
                Y, _, _ = g.generate_along(L, P, n)
            lengths = n.cpu().numpy() if hasattr(n, "cpu") else np.asarray(n)
            Tmax = int(lengths.max())
            # SSRN at the batch's longest length; rows past each utterance's length come back as 0
            _, Zd = g.engine.ssrn(Y[:, :Tmax], want_logits=False, lengths=n)
            Z = np.zeros((len(L), hp.r * hp.max_T, Zd.shape[2]), np.float32)
            Z[:, :hp.r * Tmax] = Zd.cpu().numpy()
        elif fast:
            # the whole loop on the device (CUDA-graph replay), identical results
            Y, _ = g.generate(L)
        else:
            # the reference's loop, verbatim in structure (synthesize.py:45-54)
            Y = np.zeros((len(L), hp.max_T, hp.n_mels), np.float32)
            prev_max_attentions = np.zeros((len(L),), np.int32)
            for j in range(hp.max_T):
                _gs, _Y, _max_attentions, _alignments = \
                    sess.run([g.global_step, g.Y, g.max_attentions, g.alignments],
                             {g.L: L, g.mels: Y, g.prev_max_attentions: prev_max_attentions})
                Y[:, j, :] = _Y[:, j, :]
                prev_max_attentions = _max_attentions[:, j]

        if lengths is None:
            # Get magnitude (synthesize.py:57)
            Z = sess.run(g.Z, {g.Y: Y})

    # Generate wav files (synthesize.py:60-64): Griffin-Lim on the GPU for the whole batch
    if write:
        if not os.path.exists(hp.sampledir):
            os.makedirs(hp.sampledir)
        if vocoder:
            from scipy.io.wavfile import write as write_wav
            from .utils import spectrograms2wavs
            if lengths is None:
                wavs = spectrograms2wavs(Z, momentum=momentum)
            else:
                # one call at the batch's longest length, each utterance on its own magnitude frames
                wavs = spectrograms2wavs(Z[:, :hp.r * int(lengths.max())], lengths=hp.r * lengths, momentum=momentum)
            for i, wav in enumerate(wavs):
                print("Working on file", i + 1)
                write_wav(os.path.join(hp.sampledir, "{}.wav".format(i + 1)), hp.sr, wav)
        else:
            for i, mag in enumerate(Z):
                if lengths is not None:
                    mag = mag[:hp.r * int(lengths[i])]
                np.save(os.path.join(hp.sampledir, "{}.mag.npy".format(i + 1)), mag)
    return (Y.cpu().numpy() if hasattr(Y, "cpu") else Y), Z


if __name__ == '__main__':
    synthesize()
    print("Done")
