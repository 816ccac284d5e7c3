"""Corpus aligner: every utterance of a training corpus aligned to its transcript (Engine.text2mel_align), for
per-character durations and for finding transcripts that do not match their audio.

`align_corpus` reads the corpus as the trainer does (trainer.load_train_data), sorts the utterances by text length
(stably) and aligns them B at a time, with the features from `mels/*.npy` (prepro; trainer's loader) or computed from
the wavs on the device.  It writes, under out_dir:
  alignments.tsv  one row per utterance in transcript order: fname, frames, text length, score / frames (the mean
                  log-attention along the path), and the frames of text positions 0 .. EOS, space separated; a skipped
                  utterance has its reason in the last column and "-" where no value exists;
  ranking.txt     the aligned fnames, worst first by mean log-attention: the clips to listen to first.

    python -m dc_tts_b200.align DATA_DIR OUT_DIR [--batch B] [--wavs] [--resample]

restores Text2Mel from the latest checkpoint under hp.logdir-1, and refuses to run without one."""
import argparse
import os

import numpy as np

from .hyperparams import Hyperparams as hp
from .trainer import _load_spectrograms_npy, load_train_data


def _reason(engine, text_len, frames):
    """Why an utterance cannot be aligned, or None.  frames None: not known yet."""
    h = engine.hp
    if text_len > h.max_N:
        return "text of %d characters, more than max_N = %d" % (text_len, h.max_N)
    if frames is None:
        return None
    if frames > h.max_T:
        return "%d frames, more than max_T = %d" % (frames, h.max_T)
    if text_len - 1 > (h.attention_win_size - 1) * frames:
        return "EOS at %d cannot be reached in %d frames" % (text_len - 1, frames)
    return None


def _features(engine, fpaths, from_wavs, resample, mags=False):
    """(mels (B, T_b, n_mels) zero-padded, frames (B,)) of a batch of utterances, through the trainer's loaders; with
    `mags`, also each utterance's magnitudes (B entries of (r frames_b, F), numpy or CUDA tensors) as a third value."""
    if from_wavs:
        from .utils import _read_pcm_for
        pcms, rates = zip(*[_read_pcm_for(p, resample) for p in fpaths])
        mels, mg, t, _ = engine.load_spectrograms_batch(list(pcms), rates=list(rates))
        t = np.asarray(t, np.int64)
        if mags:
            return mels, t, [mg[b, :engine.hp.r * int(t[b])] for b in range(len(t))]
        return mels, t
    loaded = [_load_spectrograms_npy(p) for p in fpaths]
    ms = [m for _, m, _ in loaded]
    t = np.array([m.shape[0] for m in ms], np.int64)
    mels = np.zeros((len(ms), max(1, int(t.max())), engine.hp.n_mels), np.float32)
    for b, m in enumerate(ms):
        mels[b, :len(m)] = m
    if mags:
        return mels, t, [g for _, _, g in loaded]
    return mels, t


def align_corpus(data_dir, engine, out_dir, B=32, prepro=None, resample=False):
    """Align every utterance of the corpus at data_dir with `engine`'s Text2Mel and write alignments.tsv and ranking.txt
    to out_dir (see the module's documentation).  `prepro` (default hp.prepro): features from mels/*.npy, else from the
    wavs on the device (`resample`: accept wavs at any sample rate).  Returns the rows, in transcript order: dicts with
    fname, text_length, frames, and either mean (score / frames) and durations or reason."""
    import torch
    fpaths, text_lengths, texts = load_train_data(data_dir)
    from_wavs = not (hp.prepro if prepro is None else prepro)
    h = engine.hp
    rows = [dict(fname=os.path.basename(p), text_length=int(n), frames=None) for p, n in zip(fpaths, text_lengths)]
    todo = []
    for i in np.argsort(text_lengths, kind="stable"):
        rows[i]["reason"] = _reason(engine, text_lengths[i], None)
        if rows[i]["reason"] is None:
            todo.append(int(i))
    for k in range(0, len(todo), B):
        batch = todo[k:k + B]
        mels, t = _features(engine, [fpaths[i] for i in batch], from_wavs, resample)
        keep = []
        for j, i in enumerate(batch):
            rows[i]["frames"] = int(t[j])
            rows[i]["reason"] = _reason(engine, text_lengths[i], int(t[j]))
            if rows[i]["reason"] is None:
                keep.append(j)
        if not keep:
            continue
        T = int(t[keep].max())
        L = np.zeros((len(keep), h.max_N), np.int32)
        for r, j in enumerate(keep):
            L[r, :len(texts[batch[j]])] = texts[batch[j]]
        sel = torch.as_tensor(keep, device=mels.device) if isinstance(mels, torch.Tensor) else keep
        m = mels[sel][:, :T]
        m = m.contiguous() if isinstance(m, torch.Tensor) else np.ascontiguousarray(m)
        _, _, dur, score = engine.text2mel_align(L, m, lengths=t[keep])
        dur, score = dur.cpu().numpy(), score.cpu().numpy()
        for r, j in enumerate(keep):
            i = batch[j]
            rows[i]["mean"] = float(score[r]) / int(t[j])
            rows[i]["durations"] = dur[r, :text_lengths[i]].tolist()
    _write(out_dir, rows)
    return rows


def _write(out_dir, rows):
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "alignments.tsv"), "w") as f:
        f.write("fname\tframes\ttext_length\tmean_log_attention\tdurations\n")
        for r in rows:
            frames = "-" if r["frames"] is None else str(r["frames"])
            if r.get("reason"):
                f.write("%s\t%s\t%d\t-\tskipped: %s\n" % (r["fname"], frames, r["text_length"], r["reason"]))
            else:
                f.write("%s\t%s\t%d\t%.6f\t%s\n" % (r["fname"], frames, r["text_length"], r["mean"],
                                                   " ".join(str(d) for d in r["durations"])))
    ranked = sorted((r for r in rows if not r.get("reason")), key=lambda r: r["mean"])
    with open(os.path.join(out_dir, "ranking.txt"), "w") as f:
        for r in ranked:
            f.write(r["fname"] + "\n")


def _restore_text2mel(engine):
    """Text2Mel from the latest checkpoint under hp.logdir-1, as synthesize restores it.  The aligner never runs SSRN;
    its variables, which a commit needs, are staged from the seeded initialiser unless they come with the checkpoint."""
    from .checkpoint import Saver, latest_checkpoint
    from .params import init_params
    ck = latest_checkpoint(hp.logdir + "-1")
    if ck is None:
        raise FileNotFoundError("no Text2Mel checkpoint under %s-1 (reference: Saver.restore(sess, None) fails)" % hp.logdir)
    engine.stage_params({k: v for k, v in init_params(0).items() if k.startswith("SSRN/")})
    Saver(var_list=["Text2Mel"]).restore(engine, ck)
    engine.commit_params()


def main(argv=None):
    ap = argparse.ArgumentParser(description="Align a corpus to its transcript with the trained Text2Mel.")
    ap.add_argument("data_dir")
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--wavs", action="store_true", help="features from the wav files on the device instead of mels/*.npy")
    ap.add_argument("--resample", action="store_true", help="with --wavs: accept wavs at any sample rate")
    a = ap.parse_args(argv)
    from .engine import get_engine
    e = get_engine()
    _restore_text2mel(e)
    rows = align_corpus(a.data_dir, e, a.out_dir, B=a.batch, prepro=not a.wavs, resample=a.resample)
    print("aligned %d of %d utterances -> %s" % (sum(1 for r in rows if not r.get("reason")), len(rows), a.out_dir))


if __name__ == "__main__":
    main()
