"""Time the linear-spectrogram path at each supported n_fft (1024 at 16 kHz, 2048 at 22.05 kHz, 4096 at 44.1 kHz):
  spectrogram2wav   32 utterances of 10.5 s (840 frames), 50 Griffin-Lim iterations
  features          one load_spectrograms_batch call on 32 ragged clips of 0.5 - 10 s
  ssrn              one Engine.ssrn pass at B = 32, T = 210, on the tensor path (16-CTA clusters at F = 2049) and on the
                    fp32 kernels
Each time is the median of --reps calls after a warm-up, CUDA events around the call.  Prints the card's name and power
limit read in the same run, then one JSON line.
   python tools/bench_sample_rates.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from dc_tts_b200.engine import Engine                # noqa: E402
from dc_tts_b200.params import init_params           # noqa: E402
from sample_rates import at_rate                     # noqa: E402

RATES = [(16000, 1024), (22050, 2048), (44100, 4096)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    res = {"card": card()}
    for sr, n_fft in RATES:
        with at_rate(sr, n_fft) as H:
            F = 1 + n_fft // 2
            e = Engine(0, hparams=H)
            e.load_params(init_params(0, "perturbed"))
            g = torch.Generator(device="cuda").manual_seed(0)
            mag = torch.rand(32, 840, F, device="cuda", generator=g) * 0.6 + 0.2
            t_voc = timed(lambda: e.spectrogram2wav(mag, n_iter=50), a.reps)
            rng = np.random.default_rng(1)
            clips = [(0.3 * rng.standard_normal(int(sr * rng.uniform(0.5, 10.0)))).astype(np.float32) for _ in range(32)]
            t_feat = timed(lambda: e.load_spectrograms_batch(clips), a.reps)
            Y = torch.rand(32, 210, H.n_mels, device="cuda", generator=g)
            e.set_tensor_path(1)
            tc_ok = e.get_option("ssrn_tc_available")
            t_ssrn_tc = timed(lambda: e.ssrn(Y, want_logits=False), a.reps)
            e.set_tensor_path(0)
            t_ssrn_fp32 = timed(lambda: e.ssrn(Y, want_logits=False), a.reps)
            e.close()
        r = dict(spectrogram2wav_ms=t_voc, load_spectrograms_batch_ms=t_feat, ssrn_tensor_ms=t_ssrn_tc,
                 ssrn_fp32_ms=t_ssrn_fp32, ssrn_tensor_path=bool(tc_ok))
        res["n_fft_%d" % n_fft] = r
        print("sr %5d n_fft %d: spectrogram2wav (32 x 10.5 s, 50 it) %.1f ms | load_spectrograms_batch (32 clips) %.1f ms | "
              "ssrn B=32 T=210 %.1f ms tensor path%s, %.1f ms fp32" % (sr, n_fft, t_voc, t_feat, t_ssrn_tc,
                                                                     "" if tc_ok else " (unavailable: fp32 kernels)",
                                                                     t_ssrn_fp32), flush=True)
    print("card:", res["card"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
