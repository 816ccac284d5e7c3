"""The trainer's samples at a checkpoint (trainer.write_samples) on a stub engine: file names, the WAV bytes of the audio
summary, and an event file whose every record read_events verifies.  No GPU."""
import os
import struct

import numpy as np
import torch
from scipy.io import wavfile

from dc_tts_b200 import summary, trainer
from dc_tts_b200.hyperparams import Hyperparams as hp


class StubEngine:
    """Deterministic stand-ins for the calls write_samples makes; records them."""

    def __init__(self):
        self.hp, self.calls = hp, []

    def refresh_synthesis(self):
        self.calls.append("refresh")

    def text2mel_generate_until(self, L, stop_pos=None, tail=0, steps=0):
        self.calls.append("generate")
        B = len(L)
        n = np.array([5, 9, hp.max_T][:B], np.int32)
        P = np.full((B, hp.max_T), -1, np.int32)
        for b in range(B):
            P[b, :n[b]] = np.minimum(np.arange(n[b]) // 2, hp.max_N - 1)
        Y = torch.rand(B, hp.max_T, hp.n_mels)
        return Y, torch.from_numpy(P), torch.from_numpy(n)

    def ssrn(self, Y, want_logits=True, lengths=None):
        self.calls.append(("ssrn", tuple(Y.shape), lengths.tolist()))
        B, T = Y.shape[:2]
        return None, torch.rand(B, hp.r * T, 1 + hp.n_fft // 2)

    def spectrogram2wav(self, mags, lengths=None, momentum=0.0):
        self.calls.append(("vocoder", tuple(mags.shape), list(np.asarray(lengths))))
        B = mags.shape[0]
        n = hp.hop_length * (np.asarray(lengths) - 1)
        wav = torch.zeros(B, int(n.max()))
        for b in range(B):
            wav[b, :n[b]] = torch.sin(torch.arange(int(n[b])) * 0.01) * 0.5
        trim = np.stack([np.zeros(B, np.int64), n], 1)
        return wav, trim


def test_sample_texts_from_list_and_file(tmp_path):
    sents = ["The birch canoe slid on the smooth planks.", "Glue the sheet to the dark blue background."]
    L = trainer.sample_texts(sents)
    f = tmp_path / "s.txt"
    f.write_text("header\n" + "".join("%d. %s\n" % (i + 1, s) for i, s in enumerate(sents)))
    assert np.array_equal(L, trainer.sample_texts(str(f)))
    assert L.shape == (2, hp.max_N)


def test_write_samples_files_and_audio_summary(tmp_path):
    eng = StubEngine()
    texts = trainer.sample_texts(["one two three.", "four five.", "six."])
    w = summary.FileWriter(str(tmp_path))
    wavs, lengths = trainer.write_samples(eng, texts, str(tmp_path), 4000, w)
    w.close()
    assert eng.calls[:2] == ["refresh", "generate"]
    assert eng.calls[2] == ("ssrn", (3, hp.max_T, hp.n_mels), [5, 9, hp.max_T])          # at the longest length
    assert list(lengths) == [5, 9, hp.max_T]
    d = tmp_path / "samples_004k"
    assert sorted(os.listdir(d)) == ["1.wav", "2.wav", "3.wav", "alignment_1.png", "alignment_2.png", "alignment_3.png"]
    for i, wav in enumerate(wavs):
        sr, data = wavfile.read(str(d / ("%d.wav" % (i + 1))))
        assert sr == hp.sr and np.array_equal(data, wav)
    events = summary.read_events(w.path)                       # verifies every record's checksums
    assert events[0]["file_version"] == "brain.Event:2"
    ev = events[1]
    assert ev["step"] == 4000
    vals = dict(ev["summary"])
    assert vals["samples/length_frames"] == np.float32(np.mean([5, 9, hp.max_T]))
    assert abs(vals["samples/eos_reached"] - 2 / 3) < 1e-6
    for i, wav in enumerate(wavs):
        a = vals["samples/%d/audio/0" % (i + 1)]
        assert a["sample_rate"] == hp.sr and a["num_channels"] == 1 and a["length_frames"] == len(wav)
        assert a["content_type"] == b"audio/wav"
        b = a["wav"]
        assert b[:4] == b"RIFF" and b[8:16] == b"WAVEfmt "
        assert struct.unpack_from("<I", b, 4)[0] == len(b) - 8
        fmt = struct.unpack_from("<HHIIHH", b, 20)
        assert fmt == (1, 1, hp.sr, 2 * hp.sr, 2, 16)
        assert b[36:40] == b"data" and struct.unpack_from("<I", b, 40)[0] == 2 * len(wav) == len(b) - 44
        pcm = np.frombuffer(b[44:], "<i2")
        assert np.array_equal(pcm, np.round(np.clip(wav, -1, 1) * 32767).astype(np.int16))


def test_write_samples_without_writer_writes_no_event(tmp_path):
    trainer.write_samples(StubEngine(), trainer.sample_texts(["a b c."]), str(tmp_path), 12000)
    assert sorted(os.listdir(tmp_path)) == ["samples_012k"]
    assert sorted(os.listdir(tmp_path / "samples_012k")) == ["1.wav", "alignment_1.png"]
