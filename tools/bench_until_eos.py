"""Time generation with each utterance ending at its text (Engine.text2mel_generate_until) against the full-length
generation, B = 32, the two alternated in one run, CUDA events, and report the frames the decode clusters executed.
Then the stages after it with the same lengths, each variant alternated with the others:
  SSRN      full at max_T frames | one ragged call at the batch's longest length | one call per utterance
  vocoder   one call over the batch at r max_T frames | one ragged call at r x the longest | one call per utterance
  chain     generate + SSRN + vocoder at full length | generate_until + ragged SSRN + ragged vocoder

SYNTHETIC LENGTHS: no trained model is available, and the seeded weights move the attention window on only ~15 % of
frames, so the EOS id is rarely reached.  The script instead sets each utterance's stop position from a full run's
window history so that its length is the available frame nearest to (ids of the Harvard sentence) x max_T / max_N.
   python tools/bench_until_eos.py [--reps 3] [--iters 5]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.data_load import eos_positions, load_data, utterance_lengths  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params, synthetic_text  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--iters", type=int, default=5)
a = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

B = 32
e = Engine(0)
e.load_params(init_params(0, "perturbed"))
ids = eos_positions(load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))) + 1
target = np.resize(np.round(ids * hp.max_T / hp.max_N).astype(int), B)
L = np.concatenate([synthetic_text(1, 100, seed=700 + b) for b in range(B)])
_, Pf, _, _ = e.text2mel_generate(L)
m = Pf.cpu().numpy()[:, 1:]
sp = np.zeros(B, np.int64)
for b in range(B):
    first = [0] + [j for j in range(1, m.shape[1]) if m[b, j] > m[b, j - 1]]
    j = min(first, key=lambda f: abs(f + 1 - target[b]))
    sp[b] = 0 if j == 0 else int(m[b, j])
lengths = utterance_lengths(m, sp, 0, steps=hp.max_T)
T_eff = int(lengths.max())
print("synthetic lengths (frames): target %s..%s, realised min %d median %d max %d" % (
    target.min(), target.max(), lengths.min(), int(np.median(lengths)), T_eff), flush=True)


def timed(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(a.iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / a.iters


runs = {
    "generate full": lambda: e.text2mel_generate(L),
    "generate until": lambda: e.text2mel_generate_until(L, stop_pos=sp),
}
for fn in runs.values():
    fn()
torch.cuda.synchronize()
res = {k: [] for k in runs}
for rep in range(a.reps):
    for k, fn in runs.items():
        res[k].append(timed(fn))
e.text2mel_generate_until(L, stop_pos=sp)
frames_until = e.get_option("decode_last_frames")
e.text2mel_generate(L)
frames_full = e.get_option("decode_last_frames")
for k, v in res.items():
    print("%-16s %s ms (median %.2f)" % (k, " ".join("%.2f" % x for x in v), float(np.median(v))), flush=True)
print("frames executed, summed over clusters: full %d, until %d" % (frames_full, frames_until), flush=True)


# ---- the stages after generation, with the same lengths ----
Y, _, n_dev = e.text2mel_generate_until(L, stop_pos=sp)
n_host = n_dev.cpu().numpy()
Yf = e.text2mel_generate(L)[0]
Zf = e.ssrn(Yf, want_logits=False)[1]
Zr = e.ssrn(Y[:, :T_eff], want_logits=False, lengths=n_dev)[1]


def ssrn_each():
    for b, k in enumerate(n_host):
        e.ssrn(Y[b:b + 1, :k], want_logits=False)


def vocoder_each(Z):
    for b, k in enumerate(n_host):
        e.spectrogram2wav(Z[b:b + 1, :hp.r * k])


def chain_full():
    Yc = e.text2mel_generate(L)[0]
    e.spectrogram2wav(e.ssrn(Yc, want_logits=False)[1])


def chain_until():
    Yc, _, nc = e.text2mel_generate_until(L, stop_pos=sp)
    Zc = e.ssrn(Yc[:, :T_eff], want_logits=False, lengths=nc)[1]
    e.spectrogram2wav(Zc, lengths=hp.r * nc.cpu().numpy())


stages = {
    "ssrn full %d" % hp.max_T: lambda: e.ssrn(Yf, want_logits=False),
    "ssrn ragged %d" % T_eff: lambda: e.ssrn(Y[:, :T_eff], want_logits=False, lengths=n_dev),
    "ssrn per utt": ssrn_each,
    "vocoder full %d" % (hp.r * hp.max_T): lambda: e.spectrogram2wav(Zf),
    "vocoder ragged %d" % (hp.r * T_eff): lambda: e.spectrogram2wav(Zr, lengths=hp.r * n_host),
    "vocoder per utt": lambda: vocoder_each(Zr),
    "chain full": chain_full,
    "chain until": chain_until,
}
for fn in stages.values():
    fn()
torch.cuda.synchronize()
res = {k: [] for k in stages}
for rep in range(a.reps):
    for k, fn in stages.items():
        res[k].append(timed(fn))
for k, v in res.items():
    print("%-20s %s ms (median %.2f)" % (k, " ".join("%.2f" % x for x in v), float(np.median(v))), flush=True)
