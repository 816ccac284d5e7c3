"""Time streaming synthesis from text (Engine.synthesis_stream) against the one-shot chain, and the decode's cost of
publishing its progress.

Texts: harvard_sentences.txt, cycled over the batch, random weights (init_params(0, "perturbed")).  Random weights do not
find the end of a text, so each utterance gets the stop position whose length is nearest to its text's share of max_T
(as tools/bench_until_eos.py does), and the decode runs until then.
  open     host clock of the open alone (allocations, TextEnc and the decode launch), and the device memory it took
           (cudaMemGetInfo before and after)
  first    host clock from the open of the stream to the return of the first poll that gave samples
  total    host clock from the open to the return of close(), against the one-shot chain text2mel_generate_until ->
           ssrn(lengths) -> spectrogram2wav(lengths) on the same texts (host clock around it, ending in a synchronise)
  underrun whether any utterance's piece arrived after the audio before it, played from the first samples at hp.sr, ran out
Decode alone: the persistent decode launch by itself, CUDA events recorded around it by the library (option
decode_timing, dctts_get_option "decode_last_us"), for generate_until (no progress) and for a stream's open (progress
published; the stream is then closed without running its chunks), each at the default utterances per cluster G and at
the stream's G (option decode_group).  The four alternate, `--reps` times each.
Every figure is the median of `--reps` repetitions after one warm-up.
   python tools/bench_synthesis_stream.py [--reps 5] [--B 1 4 32] [--chunks 8 16 32] [--decode-B 1 4 7 16 32]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.data_load import eos_positions, load_data  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--B", type=int, nargs="+", default=[1, 4, 32])
ap.add_argument("--chunks", type=int, nargs="+", default=[8, 16, 32])
ap.add_argument("--decode-B", type=int, nargs="+", default=[1, 4, 7, 16, 32])
a = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

e = Engine(0)
e.load_params(init_params(0, "perturbed"))
harvard = load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))
SR = hp.sr
print("decode_max_clusters:", e.get_option("decode_max_clusters"), flush=True)


def texts(B):
    L = harvard[np.arange(B) % len(harvard)]
    target = np.round((eos_positions(L) + 1) * hp.max_T / hp.max_N).astype(int)
    _, P, _, _ = e.text2mel_generate(L)
    m = P.cpu().numpy()[:, 1:]
    sp = np.zeros(B, np.int64)
    for b in range(B):
        first = [0] + [j for j in range(1, m.shape[1]) if m[b, j] > m[b, j - 1]]
        j = min(first, key=lambda f: abs(f + 1 - target[b]))
        sp[b] = 0 if j == 0 else int(m[b, j])
    return L, sp


def streamed(L, sp, chunk, momentum):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    ss = e.synthesis_stream(L, stop_pos=sp, chunk=chunk, momentum=momentum)
    t_open = time.perf_counter() - t0
    mem = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20
    B = len(L)
    first, ok = None, True
    played = np.zeros(B)                                   # samples each utterance has had before the current piece
    start = np.full(B, np.nan)                             # when each utterance's first samples arrived
    for out in ss:
        now = time.perf_counter()
        n = np.array([o.size for o in out])
        if first is None and n.any():
            first = now
        late = (n > 0) & (played > 0) & (played / SR < now - start)
        ok = ok and not late.any()
        start[(n > 0) & (played == 0)] = now
        played += n
    ss.close()
    return first - t0, time.perf_counter() - t0, ok, float(played.max()) / SR, t_open, mem


def one_shot(L, sp):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    Y, _, n = e.text2mel_generate_until(L, stop_pos=sp)
    _, Z = e.ssrn(Y, lengths=n, want_logits=False)
    e.spectrogram2wav(Z, lengths=4 * n.cpu().numpy())
    return time.perf_counter() - t0


def groups(B):
    """(default G, stream G): the fewest utterances per cluster that keep every cluster co-resident, and the fewest that
    leave one co-resident cluster slot free where five per cluster allow it (api_synth.cu: decode_group)."""
    mc = max(1, e.get_option("decode_max_clusters"))

    def fewest(m):
        G = 1
        while G < 5 and -(-B // G) > m:
            G += 1
        return G
    return fewest(mc), fewest(mc - 1 if mc > 1 and -(-B // 5) <= mc - 1 else mc)


def decode_us(L, sp, progress, G):
    """GPU time of the persistent decode launch alone, at G utterances per cluster."""
    e.set_option("decode_group", G)
    if progress:
        ss = e.synthesis_stream(L, stop_pos=sp, chunk=hp.max_T)
        us = e.get_option("decode_last_us")
        ss._free()
    else:
        e.text2mel_generate_until(L, stop_pos=sp)
        us = e.get_option("decode_last_us")
    e.set_option("decode_group", 0)
    return us / 1e3


rows = []
e.set_option("decode_timing", 1)
for B in a.decode_B:
    L, sp = texts(B)
    Gs = groups(B)
    cases = [(p, G) for G in sorted(set(Gs)) for p in (False, True)]
    for c in cases:
        decode_us(L, sp, *c)
    t = {c: [] for c in cases}
    for _ in range(a.reps):
        for c in cases:
            t[c].append(decode_us(L, sp, *c))
    row = dict(kind="decode", B=B, default_G=Gs[0], stream_G=Gs[1],
               ms={"%s G=%d" % ("progress" if p else "until", G): [float(np.median(v)), min(v), max(v)] for (p, G), v in t.items()})
    rows.append(row)
    print(json.dumps(row), flush=True)
e.set_option("decode_timing", 0)
for B in a.B:
    L, sp = texts(B)
    one_shot(L, sp)
    t_one = float(np.median([one_shot(L, sp) for _ in range(a.reps)]))
    for momentum in (0.0, 0.99):
        for chunk in a.chunks:
            streamed(L, sp, chunk, momentum)
            runs = [streamed(L, sp, chunk, momentum) for _ in range(a.reps)]
            row = dict(kind="stream", B=B, momentum=momentum, chunk=chunk, first_ms=1e3 * float(np.median([r[0] for r in runs])),
                       total_ms=1e3 * float(np.median([r[1] for r in runs])), one_shot_ms=1e3 * t_one,
                       no_underrun=all(r[2] for r in runs), longest_audio_s=runs[0][3],
                       open_ms=1e3 * float(np.median([r[4] for r in runs])), open_MiB=float(np.median([r[5] for r in runs])))
            rows.append(row)
            print(json.dumps(row), flush=True)
print(json.dumps(dict(card=card, rows=rows)))
e.close()
