"""Held-out evaluation: how good a checkpoint is on recordings it was not trained on.

`split_heldout` sets utterances of the corpus aside, deterministically and identically on every rank.  `HeldOut` reads
their recorded features once (mels/*.npy, or computed from the wavs on the device, as the corpus aligner does:
align._features) and `HeldOut.run` evaluates the weights the engine holds, one row per utterance in batches sorted by
text length:
  num = 1 (Text2Mel)  the free run until the EOS (Engine.text2mel_generate_until, after Engine.refresh_synthesis):
                      mel-level MCD-DTW of the generated mels against the recording's (Engine.mcd_dtw), the window checks
                      of its attention-window history (eos_reached: it stopped before max_T frames; skipped: text
                      positions before the EOS that are no frame's window; longest_stall: the most frames under one
                      window; length_ratio: generated / recorded frames), and the aligner's mean log-attention of the
                      recording (Engine.text2mel_align);
  num = 2 (SSRN)      copy synthesis, recorded mels -> SSRN -> Griffin-Lim -> the device feature extraction, and the
                      wav-level MCD-DTW of the result against the recording's mels;
and for both the teacher-forced validation losses of the training graph (trainer.evaluate) over the held-out set.
The MCD is the MFCC-style variant (DESIGN.md section 8h): its values are not comparable to published MCD figures.

    python -m dc_tts_b200.heldout DATA_DIR OUT_DIR [--list FILE] [--batch B] [--wavs] [--resample] [--num 1|2]

restores the network evaluated from the latest checkpoint under hp.logdir-1 (Text2Mel) or hp.logdir-2 (SSRN), refuses
to run without it, and writes heldout.tsv (one row per utterance) and summary.json to OUT_DIR.  `--list` names the
utterances to evaluate, one fname per line: the heldout.txt that `trainer.train(..., heldout=...)` writes."""
import argparse
import json
import os

import numpy as np

from .align import _features, _reason
from .hyperparams import Hyperparams as hp

COLUMNS = {1: ["fname", "frames", "text_length", "mcd", "pairs", "generated", "eos_reached", "skipped", "longest_stall",
               "length_ratio", "mean_log_attention", "note"],
           2: ["fname", "frames", "text_length", "mcd", "pairs", "note"]}


def split_heldout(fpaths, text_lengths, texts, n, seed=0):
    """(train, heldout): two (fpaths, text_lengths, texts) triples in load_train_data's format.  `n` utterances drawn by
    a permutation of `seed` are held out, in corpus order; the rest, also in corpus order, is for training.  The split
    depends on nothing but its arguments, so every rank of a data-parallel run draws the same one."""
    total = len(fpaths)
    if not 1 <= n < total:
        raise ValueError("split_heldout: n must be in [1, %d) for %d utterances, got %d" % (total, total, n))
    held = np.zeros(total, bool)
    held[np.random.default_rng(seed).permutation(total)[:n]] = True

    def pick(mask):
        idx = np.flatnonzero(mask)
        return [fpaths[i] for i in idx], [text_lengths[i] for i in idx], [texts[i] for i in idx]
    return pick(~held), pick(held)


def window_checks(P, n, e, t, max_T):
    """The window checks of one free run: P the window of every frame (>= n entries), n frames generated, e the EOS
    position, t the recording's frames.  Returns dict(eos_reached, skipped, longest_stall, length_ratio)."""
    w = np.asarray(P[:n], np.int64)
    skipped = int(e - np.unique(w[(w >= 0) & (w < e)]).size) if e > 0 else 0
    stall = 0
    if n > 0:
        starts = np.flatnonzero(np.concatenate([[True], w[1:] != w[:-1], [True]]))
        stall = int(np.diff(starts).max())
    return dict(eos_reached=bool(n < max_T), skipped=skipped, longest_stall=stall, length_ratio=float(n) / float(t))


def _fmt(v):
    if isinstance(v, bool):
        return "1" if v else "0"
    if isinstance(v, float):
        return "%.6f" % v
    return str(v)


def write_table(path, rows, num):
    """One line per row under COLUMNS[num]; a row set aside has "-" for every value it lacks and its reason in `note`."""
    cols = COLUMNS[num]
    with open(path, "w") as f:
        f.write("\t".join(cols) + "\n")
        for r in rows:
            vals = []
            for c in cols:
                if c == "note":
                    vals.append("skipped: " + r["reason"] if r.get("reason") else "")
                else:
                    vals.append("-" if r.get(c) is None else _fmt(r[c]))
            f.write("\t".join(vals) + "\n")


def write_summary(path, summary):
    with open(path, "w") as f:
        json.dump(summary, f, indent=1, sort_keys=True)
        f.write("\n")


def scalars(summary):
    """The summary's numbers as flat (name, value) pairs, losses as loss/<name>, in a fixed order."""
    out = [(k, float(v)) for k, v in sorted(summary.items())
           if isinstance(v, (int, float)) and not isinstance(v, bool) and k not in ("global_step", "num")]
    out += [("loss/" + k, float(v)) for k, v in sorted(summary.get("losses", {}).items())]
    return out


def append_log(path, global_step, summary):
    """A row of `scalars(summary)` at `global_step` appended to the TSV at `path` (its header written first when new)."""
    sc = scalars(summary)
    new = not os.path.exists(path)
    with open(path, "a") as f:
        if new:
            f.write("\t".join(["global_step"] + [k for k, _ in sc]) + "\n")
        f.write("\t".join([str(int(global_step))] + ["%.6f" % v for _, v in sc]) + "\n")


class HeldOut:
    """The held-out utterances and their recorded features, read once (see the module's documentation).  `prepro`
    (default hp.prepro): features from mels/*.npy and mags/*.npy, else from the wavs on the device (`resample`: accept
    wavs at any sample rate).  An utterance that cannot run -- text over max_N, recording over max_T frames, EOS not
    reachable in its frames -- is set aside with its reason, as the aligner does.  `B`: utterances per evaluation batch."""

    def __init__(self, engine, fpaths, text_lengths, texts, prepro=None, resample=False, B=32):
        if B < 1:
            raise ValueError("HeldOut: B must be >= 1")
        self.B, self.r = int(B), engine.hp.r
        self.fnames = [os.path.basename(p) for p in fpaths]
        from_wavs = not (hp.prepro if prepro is None else prepro)
        r = self.r
        self.items = [dict(fname=f, text_length=int(n), text=np.asarray(t, np.int32), frames=None, mel=None, mag=None,
                           reason=_reason(engine, int(n), None))
                      for f, n, t in zip(self.fnames, text_lengths, texts)]
        todo = [i for i in np.argsort(text_lengths, kind="stable") if self.items[i]["reason"] is None]
        for k in range(0, len(todo), self.B):
            batch = todo[k:k + self.B]
            mels, t, mags = _features(engine, [fpaths[i] for i in batch], from_wavs, resample, mags=True)
            mels = mels.cpu().numpy() if hasattr(mels, "cpu") else np.asarray(mels)
            for j, i in enumerate(batch):
                it = self.items[i]
                it["frames"] = int(t[j])
                it["reason"] = _reason(engine, it["text_length"], int(t[j]))
                if it["reason"] is None:
                    it["mel"] = np.ascontiguousarray(mels[j, :t[j]], np.float32)
                    m = mags[j]
                    it["mag"] = np.ascontiguousarray((m.cpu().numpy() if hasattr(m, "cpu") else m)[:r * t[j]], np.float32)
        # the evaluation order: text length, stably
        self.order = [i for i in np.argsort(text_lengths, kind="stable") if self.items[i]["reason"] is None]

    def _batch(self, idx, n_text=None):
        """Texts (b, n_text or the longest) and zero-padded recorded mels (b, T_b, n_mels), mags (b, r T_b, F) and frames."""
        its = [self.items[i] for i in idx]
        t = np.array([it["frames"] for it in its], np.int64)
        N = n_text or max(it["text_length"] for it in its)
        L = np.zeros((len(its), N), np.int32)
        mels = np.zeros((len(its), int(t.max()), its[0]["mel"].shape[1]), np.float32)
        mags = np.zeros((len(its), self.r * int(t.max()), its[0]["mag"].shape[1]), np.float32)
        for b, it in enumerate(its):
            L[b, :it["text_length"]] = it["text"][:it["text_length"]]
            mels[b, :it["frames"]] = it["mel"]
            mags[b, :it["mag"].shape[0]] = it["mag"]
        return L, mels, mags, t

    def run(self, engine, num, global_step, train_batch=None, K=24):
        """Evaluate the engine's weights for `num` (1: Text2Mel, 2: SSRN).  Returns (rows, summary): rows in the order the
        utterances were given, dicts with the columns of COLUMNS[num] (a row set aside has its `reason`), and the summary:
        utterances, evaluated, set_aside, mcd_mean, mcd_median, for num = 1 also eos_reached (a share), skipped_mean,
        longest_stall_mean, length_ratio_mean and mean_log_attention, and the validation losses.

        The validation losses are the training graph's (trainer.evaluate, dropout and all, without an update) on the
        held-out utterances in text-length order, in batches of exactly `train_batch` utterances (default self.B), the
        batch size the training workspace was initialised with: the last batch is completed with the first utterances
        again.  A batch beyond the workspace's capacity (Engine.train_capacity) is skipped and counted
        (loss_batches_skipped).  Nothing of the training state changes."""
        import torch
        from .data_load import eos_positions
        if num not in (1, 2):
            raise ValueError("HeldOut.run: num must be 1 (Text2Mel) or 2 (SSRN)")
        h = engine.hp
        rows = [dict(fname=it["fname"], text_length=it["text_length"], frames=it["frames"], reason=it["reason"])
                for it in self.items]
        engine.refresh_synthesis()
        for k in range(0, len(self.order), self.B):
            idx = self.order[k:k + self.B]
            L, mels, _, t = self._batch(idx, h.max_N)
            md = torch.from_numpy(mels).to(engine.device)
            if num == 1:
                Y, P, n = engine.text2mel_generate_until(L)
                nh = n.cpu().numpy()
                mcd, pairs = engine.mcd_dtw(Y, nh, md, t, K=K)
                _, _, _, score = engine.text2mel_align(L, md, lengths=t)
                P, score = P.cpu().numpy(), score.cpu().numpy()
                ends = eos_positions(L)
            else:
                from .utils import spectrograms2wavs
                _, Z = engine.ssrn(md, want_logits=False, lengths=t)
                wavs = spectrograms2wavs(Z, lengths=h.r * t, engine=engine)
                m2, _, t2, _ = engine.load_spectrograms_batch(wavs)
                t2 = np.maximum(np.asarray(t2, np.int64), 1)
                mcd, pairs = engine.mcd_dtw(m2, t2, md, t, K=K)
            mcd, pairs = mcd.cpu().numpy(), pairs.cpu().numpy()
            for b, i in enumerate(idx):
                r = rows[i]
                r["mcd"], r["pairs"] = float(mcd[b]), int(pairs[b])
                if num == 1:
                    r["generated"] = int(nh[b])
                    r.update(window_checks(P[b], int(nh[b]), int(ends[b]), int(t[b]), h.max_T))
                    r["mean_log_attention"] = float(score[b]) / int(t[b])
        summary = self._summary(rows, num)
        summary.update(self._losses(engine, num, global_step, train_batch or self.B))
        summary["global_step"] = int(global_step)
        return rows, summary

    def _losses(self, engine, num, global_step, B):
        from .trainer import evaluate
        n = len(self.order)
        if n == 0:
            return dict(losses={}, loss_batches=0, loss_batches_skipped=0)
        N_cap, T_cap = engine.train_capacity()
        sums, used, skipped = {}, 0, 0
        for k in range(0, n, B):
            idx = [self.order[(k + j) % n] for j in range(B)]
            L, mels, mags, _ = self._batch(idx)
            if mels.shape[1] > T_cap or (num == 1 and L.shape[1] > N_cap):
                skipped += 1
                continue
            losses = evaluate(num, engine, L, mels, mags, global_step)[0]
            for key, v in losses.items():
                sums[key] = sums.get(key, 0.0) + float(v)
            used += 1
        return dict(losses={key: v / used for key, v in sums.items()}, loss_batches=used, loss_batches_skipped=skipped)

    @staticmethod
    def _summary(rows, num):
        done = [r for r in rows if not r.get("reason")]
        s = dict(num=num, utterances=len(rows), evaluated=len(done), set_aside=len(rows) - len(done))
        if not done:
            return s
        mcd = np.array([r["mcd"] for r in done])
        s["mcd_mean"], s["mcd_median"] = float(mcd.mean()), float(np.median(mcd))
        if num == 1:
            s["eos_reached"] = float(np.mean([r["eos_reached"] for r in done]))
            for key in ("skipped", "longest_stall", "length_ratio", "mean_log_attention"):
                s[key + ("" if key == "mean_log_attention" else "_mean")] = float(np.mean([r[key] for r in done]))
        return s

    def write(self, out_dir, rows, summary, num):
        """heldout.tsv and summary.json under out_dir."""
        os.makedirs(out_dir, exist_ok=True)
        write_table(os.path.join(out_dir, "heldout.tsv"), rows, num)
        write_summary(os.path.join(out_dir, "summary.json"), summary)


def read_list(path):
    """The fnames of a list file (one per line, blank lines ignored)."""
    with open(path) as f:
        return [line.strip() for line in f if line.strip()]


def select(fpaths, text_lengths, texts, names):
    """The utterances of the corpus named in `names` (basenames), in corpus order; a name not in the corpus is refused."""
    want = set(names)
    have = {os.path.basename(p) for p in fpaths}
    missing = sorted(want - have)
    if missing:
        raise ValueError("%d listed utterances are not in the corpus, e.g. %s" % (len(missing), missing[0]))
    keep = [i for i, p in enumerate(fpaths) if os.path.basename(p) in want]
    return [fpaths[i] for i in keep], [text_lengths[i] for i in keep], [texts[i] for i in keep]


def parser():
    ap = argparse.ArgumentParser(description="Evaluate the latest checkpoint on held-out recordings (MCD-DTW, window "
                                             "checks, validation losses).")
    ap.add_argument("data_dir")
    ap.add_argument("out_dir")
    ap.add_argument("--list", help="evaluate only the fnames in this file (one per line), e.g. a trainer's heldout.txt")
    ap.add_argument("--batch", type=int, default=32, help="utterances per batch (also the validation losses' batch)")
    ap.add_argument("--wavs", action="store_true", help="features from the wav files on the device instead of mels/*.npy")
    ap.add_argument("--resample", action="store_true", help="with --wavs: accept wavs at any sample rate")
    ap.add_argument("--num", type=int, choices=(1, 2), default=1, help="1: Text2Mel (default), 2: SSRN")
    return ap


def _restore(engine, num):
    """The network evaluated from the latest checkpoint under hp.logdir-<num> (refused without one); the other network,
    which the evaluation never runs but a commit needs, from its checkpoint when there is one, else the seeded initialiser.
    Returns the checkpoint's global step."""
    from .checkpoint import Saver, latest_checkpoint, list_variables, load_checkpoint
    from .params import init_params
    scopes = {1: "Text2Mel", 2: "SSRN"}
    ck = latest_checkpoint(hp.logdir + "-%d" % num)
    if ck is None:
        raise FileNotFoundError("no %s checkpoint under %s-%d" % (scopes[num], hp.logdir, num))
    other = 3 - num
    ck_other = latest_checkpoint(hp.logdir + "-%d" % other)
    if ck_other is None:
        engine.stage_params({k: v for k, v in init_params(0).items() if k.startswith(scopes[other] + "/")})
    else:
        Saver(var_list=[scopes[other]]).restore(engine, ck_other)
    Saver(var_list=[scopes[num]]).restore(engine, ck)
    engine.commit_params()
    names = {v for v, _, _ in list_variables(ck)}
    return int(load_checkpoint(ck, ["gs/global_step"])["gs/global_step"]) if "gs/global_step" in names else 0


def main(argv=None):
    from .trainer import load_train_data
    a = parser().parse_args(argv)
    if a.batch < 1:
        raise SystemExit("--batch must be >= 1")
    from .checkpoint import latest_checkpoint
    if latest_checkpoint(hp.logdir + "-%d" % a.num) is None:
        raise FileNotFoundError("no %s checkpoint under %s-%d" % ({1: "Text2Mel", 2: "SSRN"}[a.num], hp.logdir, a.num))
    fpaths, text_lengths, texts = load_train_data(a.data_dir)
    if a.list:
        fpaths, text_lengths, texts = select(fpaths, text_lengths, texts, read_list(a.list))
    from .engine import get_engine
    e = get_engine()
    gs = _restore(e, a.num)
    if a.num == 1:
        e.train_init(a.batch)
    else:
        e.train_init_ssrn(a.batch, e.hp.max_T)
    held = HeldOut(e, fpaths, text_lengths, texts, prepro=not a.wavs, resample=a.resample, B=a.batch)
    rows, summary = held.run(e, a.num, gs)
    held.write(a.out_dir, rows, summary, a.num)
    print("evaluated %d of %d utterances at global step %d -> %s" % (summary["evaluated"], summary["utterances"], gs, a.out_dir))
    return summary


if __name__ == "__main__":
    main()
