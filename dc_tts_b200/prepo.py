"""Pre-computes the training targets, like the reference's prepo.py (/root/reference/prepo.py:15-25): for every wav of
the transcript, `mels/<name>.npy` (reduced mel, utils.py:147-162) and `mags/<name>.npy`.  The spectrograms come from the
GPU feature-extraction row: hp.B files per device call (`dc_tts_b200.utils.load_spectrograms_batch` ->
`dctts_load_spectrograms_batch`), each utterance's rows sliced back out of the padded batch -- the same bytes as
`utils.load_spectrograms` file by file.  Training from the wav files directly (hp.prepro = False,
trainer.bucketed_batches(..., prepro=False)) needs no pre-computation at all."""
import os

import numpy as np

from .hyperparams import Hyperparams as hp
from .trainer import load_train_data


def _save(out_dir, fname, mel, mag):
    np.save(os.path.join(out_dir, "mels", fname.replace("wav", "npy")), mel)
    np.save(os.path.join(out_dir, "mags", fname.replace("wav", "npy")), mag)


def prepo(data_dir=None, out_dir=".", load_spectrograms=None, progress=None, batch_size=None, engine=None, resample=False):
    """`load_spectrograms(fpath) -> (fname, mel, mag)`, when given, is called file by file; by default the files go to the
    device `batch_size` (hp.B) at a time.  `resample=True` accepts files at any sample rate and resamples them to hp.sr on
    the device (utils.load_spectrograms_batch); otherwise a file at another rate is refused."""
    fpaths, _, _ = load_train_data(data_dir)
    for sub in ("mels", "mags"):
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    stream = progress(fpaths) if progress else fpaths
    if load_spectrograms is not None:
        for fpath in stream:
            _save(out_dir, *load_spectrograms(fpath))
        return len(fpaths)
    batch_size = batch_size or hp.B
    chunk = []
    for fpath in stream:
        chunk.append(fpath)
        if len(chunk) == batch_size:
            _save_batch(out_dir, chunk, engine, resample)
            chunk = []
    if chunk:
        _save_batch(out_dir, chunk, engine, resample)
    return len(fpaths)


def _save_batch(out_dir, fpaths, engine, resample):
    from .utils import load_spectrograms_batch
    fnames, mels, mags, t = load_spectrograms_batch(fpaths, engine, resample)
    mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
    for b, fname in enumerate(fnames):
        _save(out_dir, fname, mels[b, :t[b]], mags[b, :hp.r * t[b]])


if __name__ == "__main__":
    print("Done", prepo())
