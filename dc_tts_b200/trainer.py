"""The trainer loop around `Engine.train_step` / `train_step_ssrn` -- what `python train.py 1|2` does in the reference
(/root/reference/train.py:137-160: one optimiser step per batch, a checkpoint `model_gs_{NNN}k` every 1000 steps in
`hp.logdir + "-" + num`, stop after hp.num_iterations) on top of the transcript parser of data_load.py:41-77 and the
pre-computed `mels/*.npy`, `mags/*.npy` of prepo.py (data_load.py:104-112), or, with hp.prepro = False, features computed
on the device from the wav files one bucket at a time.

Batching: `bucketed_batches` restates the reference's length-bucketed, dynamically padded queue (data_load.py:88-131:
shuffled stream, buckets by text length every 20 characters, a full bucket emits a batch padded to its own longest
member).  `train` and `Graph(num, mode="train")` take those batches as they are: the CUDA step runs at each batch's own
(N_b, T_b), up to the capacity (hp.max_N, hp.max_T), and its losses are the reference's at that shape.  A batch beyond
the capacity is skipped and counted by default (`beyond_capacity="skip"`); with `beyond_capacity="grow"` the workspace
grows in place to take it, as the reference trains every batch whatever its shape, and the optimiser state is kept
(`Capacity`).  `fixed_size_batches` (plain shuffled batches padded to (max_N, max_T), BASELINE
config 5) and `pad_to_fixed` (a bucket padded further to the fixed shapes) remain for fixed-shape training.
"""
import codecs
import os
import time

import numpy as np

from .data_load import load_vocab, text_normalize
from .hyperparams import Hyperparams as hp


def _text_ids(char2idx, text, transcript, lineno):
    """`[char2idx[char] for char in text]` (data_load.py:54,73); a character outside hp.vocab raises, naming the line."""
    try:
        return np.array([char2idx[ch] for ch in text], np.int32)
    except KeyError as e:
        raise ValueError("%s:%d: character %r is not in hp.vocab" % (transcript, lineno, e.args[0])) from None


def load_train_data(data_dir=None):
    """data_load.py:41-77: transcript.csv -> (wav paths, text lengths, int32 id arrays ending in E).  As in the reference,
    a data path containing "LJ" is LJ Speech (`fname|raw|text`, wavs/<fname>.wav, text normalised); any other is the
    five-field format of its other corpora (`fname|raw|text|is_inside_quotes|duration`, the path joined to fname as is,
    no normalisation, clips longer than 10 s skipped)."""
    data_dir = data_dir or hp.data
    char2idx, _ = load_vocab()
    transcript = os.path.join(data_dir, "transcript.csv")
    lj = "LJ" in data_dir
    fpaths, text_lengths, texts = [], [], []
    for lineno, line in enumerate(codecs.open(transcript, "r", "utf-8").readlines(), 1):
        if lj:
            fname, _, text = line.strip().split("|")
            fpath, text = os.path.join(data_dir, "wavs", fname + ".wav"), text_normalize(text)
        else:
            fname, _, text, _, duration = line.strip().split("|")
            if float(duration) > 10.:
                continue
            fpath = os.path.join(data_dir, fname)
        ids = _text_ids(char2idx, text + "E", transcript, lineno)
        fpaths.append(fpath)
        text_lengths.append(len(ids))
        texts.append(ids)
    return fpaths, text_lengths, texts


def _load_spectrograms_npy(fpath, mels_dir="mels", mags_dir="mags"):
    """data_load.py:105-109: what prepo.py wrote for this wav."""
    fname = os.path.basename(fpath)
    return fname, np.load(os.path.join(mels_dir, fname.replace("wav", "npy"))), np.load(os.path.join(mags_dir, fname.replace("wav", "npy")))


def fixed_size_batches(fpaths, texts, B=None, seed=0, loader=_load_spectrograms_npy, epochs=None, rank=0, world=1):
    """Shuffled batches of exactly B utterances, zero-padded to (B, max_N), (B, max_T, n_mels), (B, 4 max_T, F).
    Utterances that do not fit are skipped; an incomplete last batch of an epoch is dropped (num_batch = len // B,
    data_load.py:97).  Data-parallel runs: every rank draws the SAME permutation (same seed) and keeps every
    world-th utterance, so the ranks' batches are disjoint."""
    B = B or hp.B
    F = 1 + hp.n_fft // 2
    rng = np.random.default_rng(seed)
    epoch = 0
    while epochs is None or epoch < epochs:
        yielded = 0
        order = rng.permutation(len(fpaths))[rank::world]
        L = np.zeros((B, hp.max_N), np.int32)
        mels = np.zeros((B, hp.max_T, hp.n_mels), np.float32)
        mags = np.zeros((B, hp.max_T * hp.r, F), np.float32)
        names, n = [], 0
        for i in order:
            text = texts[i]
            if len(text) > hp.max_N:
                continue
            fname, mel, mag = loader(fpaths[i])
            if mel.shape[0] > hp.max_T or mag.shape[0] > hp.max_T * hp.r:
                continue
            L[n, :len(text)] = text
            mels[n, :mel.shape[0]] = mel
            mags[n, :mag.shape[0]] = mag
            names.append(fname)
            n += 1
            if n == B:
                yield L, mels, mags, names
                yielded += 1
                L = np.zeros_like(L); mels = np.zeros_like(mels); mags = np.zeros_like(mags)
                names, n = [], 0
        if yielded == 0:                          # ADVICE r1: never spin forever re-reading a data set that cannot fill a batch
            raise ValueError("fixed_size_batches: fewer than B=%d utterances fit max_N=%d / max_T=%d (of %d)"
                             % (B, hp.max_N, hp.max_T, len(fpaths)))
        epoch += 1


def bucket_boundaries(text_lengths):
    """data_load.py:125: `[i for i in range(minlen + 1, maxlen - 1, 20)]`."""
    return list(range(min(text_lengths) + 1, max(text_lengths) - 1, 20))


def bucket_index(length, boundaries):
    """tf.contrib.training.bucket_by_sequence_length: bucket k holds boundaries[k-1] <= length < boundaries[k]
    (bucket 0: length < boundaries[0]; the last bucket: length >= boundaries[-1])."""
    return int(np.searchsorted(np.asarray(boundaries), length, side="right"))


def _pad_spectrograms(items):
    """dynamic_pad (data_load.py:128) of the npy route: [(mel, mag), ...] -> zero-padded (mels, mags) numpy arrays."""
    T_b = max(m.shape[0] for m, _ in items)
    Tm_b = max(g.shape[0] for _, g in items)
    mels = np.zeros((len(items), T_b, hp.n_mels), np.float32)
    mags = np.zeros((len(items), Tm_b, items[0][1].shape[1]), np.float32)
    for b, (m, g) in enumerate(items):
        mels[b, :m.shape[0]] = m; mags[b, :g.shape[0]] = g
    return mels, mags


def bucketed_batches(fpaths, text_lengths, texts, B=None, seed=0, loader=_load_spectrograms_npy, epochs=None, rank=0, world=1,
                     prepro=None, engine=None, features=None, resample=False):
    """The reference's input pipeline (data_load.py:88-131) without TensorFlow queues: a shuffled stream of utterances
    (slice_input_producer :99) is routed by TEXT length into buckets (boundaries :125); a bucket that has collected B
    utterances emits them as one batch, every tensor padded with zeros to the longest member of THAT batch
    (dynamic_pad=True, :128): L (B, N_b) int32, mels (B, T_b, n_mels), mags (B, 4 T_b', F).  Buckets keep their partial
    contents across epochs like the TF queue does; nothing is dropped except what never fills a bucket.
    Yields (L, mels, mags, names, bucket), which `train` and `Graph(mode="train")` take directly.  Data-parallel runs:
    like fixed_size_batches, every rank draws the SAME permutation (same seed) and keeps every world-th utterance, so the
    ranks' batches are disjoint (their shapes may differ from rank to rank).

    `prepro` (default hp.prepro) picks where the spectrograms come from, as in data_load.py:104-113.  True: `loader`
    reads what prepo.py wrote (numpy batches).  False: the buckets collect the wav files' samples and native sample
    rates, and a full bucket gets its features from ONE batched device call, `features(pcms) -> (mels, mags)` when every
    file is at hp.sr and `features(pcms, rates)` otherwise (default `(engine or get_engine()).load_spectrograms_batch`,
    which resamples to hp.sr on the device first), so mels and mags are CUDA tensors and no mels/ or mags/ directory is
    needed.  A file at another rate than hp.sr is refused unless `resample=True` (a corpus at 16, 44.1 or 48 kHz).  The features run on the caller's thread (an engine handle is not thread-safe).  Routing,
    sharding and padding are the same loop for both routes."""
    B = B or hp.B
    from_wavs = not (hp.prepro if prepro is None else prepro)
    if from_wavs:
        from .utils import _read_pcm_for
        if features is None:
            def features(pcms, rates=None):
                from .engine import get_engine
                return (engine or get_engine()).load_spectrograms_batch(pcms, rates=rates)[:2]
    bounds = bucket_boundaries(text_lengths)
    pending = [[] for _ in range(len(bounds) + 1)]
    rng = np.random.default_rng(seed)
    epoch = 0
    while epochs is None or epoch < epochs:
        emitted = 0
        for i in rng.permutation(len(fpaths))[rank::world]:
            k = bucket_index(text_lengths[i], bounds)
            if from_wavs:
                pending[k].append((texts[i], _read_pcm_for(fpaths[i], resample), os.path.basename(fpaths[i])))
            else:
                fname, mel, mag = loader(fpaths[i])
                pending[k].append((texts[i], (mel, mag), fname))
            if len(pending[k]) == B:
                items, pending[k] = pending[k], []
                L = np.zeros((B, max(len(t) for t, _, _ in items)), np.int32)
                for b, (t, _, _) in enumerate(items):
                    L[b, :len(t)] = t
                if not from_wavs:
                    mels, mags = _pad_spectrograms([it[1] for it in items])
                else:
                    pcms, rates = [it[1][0] for it in items], [it[1][1] for it in items]
                    mels, mags = features(pcms) if all(r == hp.sr for r in rates) else features(pcms, rates)
                emitted += 1
                yield L, mels, mags, [it[2] for it in items], k
        if emitted == 0 and epochs is None and epoch >= 64:
            raise ValueError("bucketed_batches: no bucket reaches B=%d utterances" % B)
        epoch += 1


def pad_to_fixed(L, mels, mags):
    """A bucketed batch in the fixed shapes of BASELINE config 5 ((B, max_N), (B, max_T, n_mels), (B, 4 max_T, F)),
    or None when the bucket is longer than those.  Zero padding is what dynamic_pad already appended, just further.
    (The trainers take bucketed batches directly; padding changes the losses, see DESIGN.md 8e.)"""
    B, N_b = L.shape
    T_b, Tm_b = mels.shape[1], mags.shape[1]
    if N_b > hp.max_N or T_b > hp.max_T or Tm_b > hp.max_T * hp.r:
        return None
    Lf = np.zeros((B, hp.max_N), np.int32); Lf[:, :N_b] = L
    mf = np.zeros((B, hp.max_T, mels.shape[2]), np.float32); mf[:, :T_b] = mels
    gf = np.zeros((B, hp.max_T * hp.r, mags.shape[2]), np.float32); gf[:, :Tm_b] = mags
    return Lf, mf, gf


def checkpoint_name(logdir, gs):
    """train.py:152."""
    return os.path.join(logdir, "model_gs_{}".format(str(gs // 1000).zfill(3) + "k"))


def over_capacity(num, L, mels, cap=hp):
    """True when a batch does not fit the training workspace: Text2Mel N_b > max_N or T_b > max_T, SSRN T_b > max_T."""
    return mels.shape[1] > cap.max_T or (num == 1 and L.shape[1] > cap.max_N)


def _round64(n):
    return -(-int(n) // 64) * 64


class Capacity:
    """The (N, T) the training workspace holds and what happens to a batch beyond it, for `train` and
    `Graph(mode="train")`.  It starts at (hp.max_N, hp.max_T), or at `capacity` = (N, T) where that is larger, which is
    reserved once right after the engine's train_init (a user who knows the corpus's longest text and clip grows the
    workspace once, up front).  `beyond_capacity`:
      "skip"  (default) a batch beyond the capacity is skipped and counted: `admit` returns False;
      "grow"  the workspace grows to the batch's shape, each growing dimension rounded up to a multiple of 64 so that a
              stream of buckets does not re-allocate at every slightly longer batch; the growth is logged and the batch
              trained.  Engine.train_reserve keeps the variables, the Adam moments and the gradient arena, so nothing of
              the optimiser is lost, and data-parallel ranks may grow at different steps.
    Past (hp.max_N, hp.max_T) the guided-attention loss covers the (max_N, max_T) table's corner only, as train.py:91-95
    crops it; the mel losses cover the whole batch."""

    def __init__(self, num, cap=hp, beyond_capacity="skip", capacity=None):
        if beyond_capacity not in ("skip", "grow"):
            raise ValueError("beyond_capacity: 'skip' or 'grow', got %r" % (beyond_capacity,))
        self.num, self.mode, self.cap = num, beyond_capacity, cap
        self.N, self.T = cap.max_N, cap.max_T
        self.requested = None
        if capacity is not None:
            N, T = (int(x) for x in capacity)
            if N < 1 or T < 1:
                raise ValueError("capacity: (N, T) >= 1, got %r" % (capacity,))
            self.requested = (N, T)
            self.N, self.T = max(self.N, N), max(self.T, T)
        self.skipped = 0

    def fits(self, L, mels):
        return mels.shape[1] <= self.T and (self.num != 1 or L.shape[1] <= self.N)

    def _reserve(self, engine):
        engine.train_reserve(self.N if self.num == 1 else 0, self.T)

    def admit(self, L, mels, log):
        """False (logged and counted) when the batch is beyond the capacity and beyond_capacity is "skip"."""
        if self.mode == "grow" or self.fits(L, mels):
            return True
        self.skipped += 1
        if self.requested is None:
            log("skipped a batch of shape N=%d, T=%d beyond the capacity (max_N=%d, max_T=%d); %d skipped so far"
                % (L.shape[1], mels.shape[1], self.cap.max_N, self.cap.max_T, self.skipped))
        else:
            log("skipped a batch of shape N=%d, T=%d beyond the capacity (N=%d, T=%d); %d skipped so far"
                % (L.shape[1], mels.shape[1], self.N, self.T, self.skipped))
        return False

    def initialised(self, engine):
        """Right after the engine's train_init: reserve the requested capacity."""
        if self.requested is not None and (self.N, self.T) != (self.cap.max_N, self.cap.max_T):
            self._reserve(engine)

    def prepare(self, engine, L, mels, log):
        """Before a step on an admitted batch: grow the workspace when the batch does not fit it."""
        if self.fits(L, mels):
            return
        if self.num == 1 and L.shape[1] > self.N:
            self.N = _round64(L.shape[1])
        if mels.shape[1] > self.T:
            self.T = _round64(mels.shape[1])
        self._reserve(engine)
        if self.num == 1:
            log("grew the training workspace to N=%d, T=%d for a batch of shape N=%d, T=%d"
                % (self.N, self.T, L.shape[1], mels.shape[1]))
        else:
            log("grew the training workspace to T=%d for a batch of T=%d" % (self.T, mels.shape[1]))


# The dropout seed of evaluations of the training graph (summaries, alignment plots).  Steps use the global step, times the
# world size plus the rank in data-parallel runs, which stays far below it.
EVAL_SEED = 0xffffffff


def evaluate(num, engine, L, mels, mags, global_step, alignments=False):
    """One forward-only evaluation of the training graph on a batch, with dropout and no update (Engine.train_eval /
    train_eval_ssrn): returns (losses, CUDA tensors Y [+ alignments] or Z, the merged Summary bytes of train.py's
    summaries with lr at `global_step`)."""
    from .summary import train_summary
    from .utils import learning_rate_decay
    if num == 1:
        losses, t = engine.train_eval(L, mels, seed=EVAL_SEED, want=("Y", "alignments") if alignments else ("Y",))
        target, out = mels, t["Y"]
    else:
        losses, t = engine.train_eval_ssrn(mels, mags, seed=EVAL_SEED)
        target, out = mags, t["Z"]
    host = lambda x: x[:1].cpu().numpy() if hasattr(x, "cpu") else np.asarray(x[:1])
    return losses, t, train_summary(num, losses, host(target), host(out), learning_rate_decay(hp.lr, global_step))


def sample_texts(samples):
    """`samples` -> (B, max_N) int32 ids through data_load.load_data("synthesize", ...): the path of a sentences file in
    harvard_sentences.txt's format (a header line, then "N. sentence" lines), or a list of sentences."""
    import tempfile
    from .data_load import load_data
    if isinstance(samples, (str, os.PathLike)):
        return load_data("synthesize", os.fspath(samples))
    samples = list(samples)
    if not samples:
        raise ValueError("samples: no sentences")
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "samples.txt")
        with codecs.open(path, "w", "utf-8") as f:
            f.write("samples\n" + "".join("%d. %s\n" % (i + 1, t.replace("\n", " ")) for i, t in enumerate(samples)))
        return load_data("synthesize", path)


def write_samples(engine, texts, logdir, global_step, writer=None):
    """What the model being trained says when it runs free, for the checkpoint at `global_step`: the engine's synthesis is
    refreshed from its current variables (Engine.refresh_synthesis), `texts` (B, max_N) are decoded until their EOS
    (Engine.text2mel_generate_until), SSRN runs on each utterance's own frames and Griffin-Lim turns them into
    `samples_{NNN}k/{i}.wav` (i from 1) in `logdir`, beside `samples_{NNN}k/alignment_{i}.png`: the attention window of
    every frame (the decode's argmax history, max_N x length).  Text2Mel and SSRN are the weights the engine holds: one of
    them is being trained, the other is as it was loaded.  With a `writer` (summary.FileWriter) one event at
    `global_step` holds an audio summary per sample (`samples/{i}/audio/0`), the mean length in frames
    (`samples/length_frames`) and the share of samples that stopped at their text's end before max_T frames
    (`samples/eos_reached`).  Returns (wavs, lengths in mel frames)."""
    from scipy.io.wavfile import write as write_wav
    from .data_load import eos_positions
    from .utils import plot_alignment, spectrograms2wavs
    h = engine.hp
    engine.refresh_synthesis()
    Y, P, n = engine.text2mel_generate_until(texts)
    lengths = n.cpu().numpy()
    Tmax = int(lengths.max())
    _, Z = engine.ssrn(Y[:, :Tmax], want_logits=False, lengths=n)
    wavs = spectrograms2wavs(Z, lengths=h.r * lengths, engine=engine)
    out = os.path.join(logdir, "samples_" + str(global_step // 1000).zfill(3) + "k")
    os.makedirs(out, exist_ok=True)
    P = P.cpu().numpy()
    for i, wav in enumerate(wavs):
        write_wav(os.path.join(out, "{}.wav".format(i + 1)), h.sr, wav)
        path = np.zeros((h.max_N, int(lengths[i])), np.float32)
        path[P[i, :lengths[i]], np.arange(lengths[i])] = 1.0
        plot_alignment(path, i + 1, out)
    if writer is not None:
        from .summary import audio, merge, scalar
        stopped = np.mean((lengths < h.max_T) & (eos_positions(np.asarray(texts)) >= 0))
        writer.add_summary(merge(*[audio("samples/%d" % (i + 1), w, h.sr) for i, w in enumerate(wavs)],
                                 scalar("samples/length_frames", float(lengths.mean())), scalar("samples/eos_reached", stopped)),
                           global_step)
        writer.flush()
    return wavs, lengths


def write_heldout(engine, heldout, num, logdir, global_step, train_batch, writer=None):
    """`heldout.run` at `global_step`: its summary appended to `logdir/heldout.tsv`, its rows in
    `heldout_{NNN}k.tsv`, and with a `writer` one event of `heldout/...` scalars.  Returns (rows, summary)."""
    from . import heldout as ho
    rows, summary = heldout.run(engine, num, global_step, train_batch=train_batch)
    ho.write_table(os.path.join(logdir, "heldout_" + str(global_step // 1000).zfill(3) + "k.tsv"), rows, num)
    ho.append_log(os.path.join(logdir, "heldout.tsv"), global_step, summary)
    if writer is not None:
        from .summary import merge, scalar
        writer.add_summary(merge(*[scalar("heldout/" + k, v) for k, v in ho.scalars(summary)]), global_step)
        writer.flush()
    return rows, summary


def train(num, engine, batches, num_iterations=None, logdir=None, global_step=None, save_every=1000, log=print, resume=True,
          rank=0, world=1, allreduce=None, beyond_capacity="skip", capacity=None, summaries=False, summary_secs=120,
          samples=None, deterministic=None, heldout=None):
    """train.py:137-160 for num = 1 (Text2Mel) or 2 (SSRN).  `batches` yields (L, mels, mags, names, ...): the bucketed
    batches of `bucketed_batches` at their own shapes or fixed-size ones; `engine` is an `Engine` with parameters loaded.
    The workspace is allocated for the capacity (hp.max_N, hp.max_T), or `capacity` = (N, T) when that is larger; a batch
    beyond it is skipped and counted in the log, or with `beyond_capacity="grow"` the workspace grows in place (keeping the
    Adam state) and the batch is trained (see `Capacity`).  Like tf.train.Supervisor (train.py:144), a `logdir` that already holds a checkpoint
    is RESUMED: variables, Adam slots and the global step come back from it (`resume=False` or an explicit `global_step`
    starts over).  Data parallel (BASELINE config 5, `world` > 1): every rank feeds its own disjoint `batches`, the step
    runs with apply=False, `allreduce` (default dc_tts_b200.parallel.allreduce_mean_) averages the flat gradient arena,
    every rank applies the identical Adam update, dropout masks differ per rank (seed = gs * world + rank) and only rank 0
    writes checkpoints.

    `summaries=True` adds what the reference's Supervisor and train.py:154-157 write, on rank 0: every `summary_secs`
    seconds of wall clock (0: after every step), at a step boundary, the next batch of `batches` is evaluated without an
    update (`evaluate`) and one event with train.py's merged summaries, `lr` and `global_step/sec` goes to a new
    `events.out.tfevents.*` file in `logdir`; at every checkpoint of Text2Mel the next batch is evaluated and its first
    alignment written as `alignment_{NNN}k.png` (utils.plot_alignment).  Evaluations consume batches as TF's queue does.

    `samples` (default None: off): sentences -- a list, or a file in harvard_sentences.txt's format -- that rank 0 synthesises
    at every checkpoint from the weights being trained (`write_samples`: wavs and window-path plots in
    `samples_{NNN}k/`, and with `summaries` an event with their audio).  The network not being trained is the one the
    engine holds: for num = 1, SSRN as loaded (e.g. restored from logdir-2; random SSRN weights still give the mels'
    lengths and a rough sound); for num = 2, Text2Mel as loaded.  It consumes no batch.
    `deterministic=True` sets the engine's option "train_deterministic" (include/dctts.h): every sum of the step runs in a
    fixed order, so a run with the same seed, data and hyper-parameters repeats bit for bit, and a run resumed from a
    checkpoint writes the bundles of the run that never stopped.  Each rank's gradient arena is deterministic; the order of
    the cross-rank all-reduce belongs to torch.distributed.  `deterministic=False` sets the option to 0 (the default
    kernels); None (the default) leaves the engine's option as it is, which is 0 unless the caller set it.
    `heldout` (default None: off): a heldout.HeldOut that rank 0 runs at every checkpoint, after the save and the samples,
    on the weights being trained.  `logdir/heldout.txt` lists its fnames (for `python -m dc_tts_b200.heldout --list`);
    each checkpoint appends the global step and the summary to `logdir/heldout.tsv` and writes the per-utterance table to
    `heldout_{NNN}k.tsv`, and with `summaries` one event holds its numbers as `heldout/...` scalars.  It consumes no
    batch and changes no training state.
    Returns the final global step."""
    if num not in (1, 2):
        raise ValueError("num: 1 for Text2Mel, 2 for SSRN (train.py:139)")
    if deterministic is not None:
        engine.set_option("train_deterministic", 1 if deterministic else 0)
    num_iterations = hp.num_iterations if num_iterations is None else num_iterations
    logdir = logdir or (hp.logdir + "-" + str(num))
    os.makedirs(logdir, exist_ok=True)
    gs = int(global_step or 0)
    cap = getattr(engine, "hp", hp)
    capa = Capacity(num, cap, beyond_capacity, capacity)
    initialised = False
    batches = iter(batches)
    writer = None
    texts = sample_texts(samples) if samples is not None and rank == 0 else None
    if heldout is not None and rank == 0:
        with open(os.path.join(logdir, "heldout.txt"), "w") as f:
            f.write("".join(n + "\n" for n in heldout.fnames))

    def next_admitted():
        for b in batches:
            if capa.admit(b[0], b[1], log):
                return b
        return None

    def evaluate_next(alignments=False):
        """`evaluate` on the next admitted batch, or None when the input pipeline is exhausted."""
        b = next_admitted()
        if b is None:
            return None
        capa.prepare(engine, b[0], b[1], log)
        return evaluate(num, engine, b[0], b[1], b[2], gs, alignments)

    while True:
        batch = next_admitted()
        if batch is None:
            break
        L, mels, mags = batch[:3]
        if not initialised:
            if num == 1:
                engine.train_init(len(L))
            else:
                engine.train_init_ssrn(len(L), cap.max_T)
            if resume and global_step is None:
                restored = engine.restore_training(logdir, "Text2Mel" if num == 1 else "SSRN")
                if restored is not None:
                    gs = restored
                    log("resumed from %s at global step %d" % (logdir, gs))
            capa.initialised(engine)
            initialised = True
            if summaries and rank == 0:
                from .summary import FileWriter, merge, scalar
                writer = FileWriter(logdir)
                last_t, last_gs = time.time(), gs
        capa.prepare(engine, L, mels, log)
        if world > 1:
            if allreduce is None:
                from .parallel import allreduce_mean_ as allreduce
            seed = gs * world + rank
            if num == 1:
                losses = engine.train_step(L, mels, global_step=gs, seed=seed, apply=False)
            else:
                losses = engine.train_step_ssrn(mels, mags, global_step=gs, seed=seed, apply=False)
            allreduce(engine.train_grads())
            engine.train_apply(gs)
        elif num == 1:
            losses = engine.train_step(L, mels, global_step=gs, seed=gs)
        else:
            losses = engine.train_step_ssrn(mels, mags, global_step=gs, seed=gs)
        gs += 1                                   # apply_gradients(..., global_step=...) increments (train.py:131)
        if gs % save_every == 0 and rank == 0:    # train.py:151-152
            engine.save_checkpoint(checkpoint_name(logdir, gs), gs, "Text2Mel" if num == 1 else "SSRN")
            log("step %d  %s" % (gs, "  ".join("%s %.4f" % kv for kv in sorted(losses.items()))))
            if writer is not None and num == 1:   # train.py:154-157
                ev = evaluate_next(alignments=True)
                if ev is not None:
                    from .utils import plot_alignment
                    plot_alignment(ev[1]["alignments"][0].cpu().numpy(), str(gs // 1000).zfill(3) + "k", logdir)
            if texts is not None:
                write_samples(engine, texts, logdir, gs, writer)
            if heldout is not None:
                write_heldout(engine, heldout, num, logdir, gs, len(L), writer)
        if writer is not None and time.time() - last_t >= summary_secs:
            ev = evaluate_next()
            now = time.time()
            if ev is not None:
                rate = (gs - last_gs) / max(now - last_t, 1e-9)
                writer.add_summary(merge(ev[2], scalar("global_step/sec", rate)), gs)
                writer.flush()
            last_t, last_gs = now, gs
        if gs > num_iterations:                   # train.py:160
            break
    if writer is not None:
        writer.close()
    return gs
