#!/usr/bin/env python
"""bench.py -- mel-frames/sec through Text2Mel (AR, 210 steps) + SSRN on N H100s.

Workload (BASELINE.json config 4 per-GPU shard; config.workload names it): every rank
synthesises `--batch` (default 32) synthetic 100-character utterances: TextEnc once, the 210
autoregressive frames in ONE persistent cluster kernel (`--decode-mode 0`: one CUDA graph per
frame, the round-1 loop), SSRN mel->linear; rank 0 receives the finished spectrograms of all ranks
in ONE NCCL gather whose chunks leave under the SSRN.  A "step" is one such pass.
`value` = N * batch * 210 * K / time, inputs resident in HBM; `e2e` = same metric through
dctts_synthesize_host (host buffers, H2D + D2H inside the timed region).

`--impl reference` times the oracle restatement of the reference's own schedule
(synthesize.py:45-57: one full-graph pass per mel frame, then SSRN) on the host cores --
the TF1 reference itself cannot run here (see DESIGN.md).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "mel_frames_per_sec"
UNIT = "mel-frames/s"


def measured_peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return dict(hbm_gbs=p["hbm_gbs"], tf=p["bf16_tflops"], tf_sustained=p.get("bf16_tflops_sustained"), src="measured")
    except Exception:
        # NVIDIA H100 SXM data sheet (700 W card): HBM3 bandwidth, dense FP16 tensor rate -- not measured here
        return dict(hbm_gbs=3350.0, tf=989.0, tf_sustained=None, src="fallback (H100 SXM data sheet)")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx, self.proc, self.lines = gpu_index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=lambda: self.lines.extend(self.proc.stdout), daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def stop(self):
        if not self.proc:
            return dict(sm_mhz=None, sm_max_mhz=None, reasons=["nvidia-smi unavailable"])
        time.sleep(0.25)
        self.proc.terminate()
        self.t.join(2)
        sm, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx = float(f[2])
            except ValueError:
                continue
            for n, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return dict(sm_mhz=(sm[len(sm) // 2] if sm else None), sm_max_mhz=mx, reasons=sorted(reasons),
                    samples=len(sm))


def usable_cores():
    """Host cores this process may really use: CPU affinity capped by the cgroup quota
    (a 128-thread pool on a quota-limited container is slower than 8 threads)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(float(txt[0]) / float(txt[1]) + 0.5)))
            else:
                q = int(txt[0])
                if q > 0:
                    per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                    n = min(n, max(1, int(q / per + 0.5)))
            break
        except Exception:
            continue
    return max(1, min(n, 32))       # torch-CPU conv/GEMM at these sizes stops scaling well before 32 threads


# ------------------------------------------------------------------------------ reference arm
def cpu_reference(passes, B=1, n_chars=100, threads=None, ssrn=True):
    """Oracle restatement of the reference schedule on the host cores: `passes` full-graph
    Text2Mel passes (each yields ONE mel frame per utterance: synthesize.py:48-53) and one
    SSRN pass, extrapolated to a 210-frame utterance."""
    import numpy as np
    import torch
    from dc_tts_b200.hyperparams import Hyperparams as hp
    from dc_tts_b200.params import init_params, synthetic_text
    from oracle import ref_torch as rt
    threads = threads or usable_cores()
    torch.set_num_threads(threads)
    P = {k: torch.from_numpy(v) for k, v in init_params(0, "perturbed").items()}
    L = synthetic_text(B, n_chars, seed=0)
    Y = torch.zeros((B, hp.max_T, hp.n_mels))
    pma = torch.zeros((B,), dtype=torch.int64)
    with torch.no_grad():
        rt.text2mel_forward(P, L, Y, pma)                      # warm-up
        t0 = time.perf_counter()
        for j in range(passes):
            o = rt.text2mel_forward(P, L, Y, pma)
            Y[:, j] = o["Y"][:, j]; pma = o["max_attentions"][:, j]
        t_pass = (time.perf_counter() - t0) / passes
        t_ssrn = 0.0
        if ssrn:
            t0 = time.perf_counter()
            rt.SSRN(P, Y)
            t_ssrn = time.perf_counter() - t0
    t_utt = hp.max_T * t_pass + t_ssrn
    return dict(value=B * hp.max_T / t_utt, t_pass=t_pass, t_ssrn=t_ssrn, cores=threads, B=B,
                # what ONE full-graph pass + SSRN would give (a schedule without the reference's O(T^2) recompute)
                single_pass_value=B * hp.max_T / (t_pass + t_ssrn),
                sample="B=%d: %d of 210 full-graph Text2Mel passes (%.3f s each) + 1 SSRN pass (%.3f s), "
                       "extrapolated to 210 passes" % (B, passes, t_pass, t_ssrn))


def cpu_baseline_block(args):
    """cpu_baseline of the bench line: the oracle at the benchmark's own batch (B = 32) and, for separating the batch
    factor from the schedule factor, at B = 1; the single-pass figures show the reference's O(T^2) factor."""
    big = cpu_reference(passes=max(1, args.cpu_passes), B=args.batch, n_chars=args.nchars)
    one = cpu_reference(passes=max(4, 4 * args.cpu_passes), B=1, n_chars=args.nchars)
    return {"value": big["value"], "unit": UNIT, "cores": big["cores"], "kind": "port", "sample": big["sample"],
            "b1": {"value": one["value"], "sample": one["sample"]},
            "single_pass_schedule": {"value_b%d" % args.batch: big["single_pass_value"], "value_b1": one["single_pass_value"],
                                     "note": "one full-graph pass + SSRN per utterance batch instead of 210 passes: what the "
                                             "reference's O(T^2) recompute costs it (x%.0f)" % (big["single_pass_value"] / big["value"])}}


def run_reference(args, rank, world):
    if rank != 0:
        return
    t0 = time.perf_counter()
    # a bench "step" of this arm = ONE full-graph pass at the benchmark batch: a bounded sample -- the reference needs 210 of
    # them (+ SSRN) per batch, which is what `value` extrapolates to
    passes = max(1, min(30, args.steps))
    r = cpu_reference(passes=passes, B=args.batch, n_chars=args.nchars)
    wall = time.perf_counter() - t0
    line = {"impl": "reference", "metric": METRIC, "value": r["value"], "unit": UNIT, "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * r["t_pass"], "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args, world),
            "cpu_baseline": {"value": r["value"], "unit": UNIT, "cores": r["cores"], "kind": "port",
                             "sample": r["sample"]},
            "e2e": {"value": r["value"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "note": "TF1 reference cannot run (no TensorFlow; tf.contrib needs TF1/py<=3.7): timed the oracle "
                    "restatement (torch-CPU fp32) of synthesize.py's own O(T^2) schedule at the benchmark batch "
                    "(B=%d per GPU; ONE host, so at N GPUs the ratio divides N shards by one CPU run); wall %.1f s"
                    % (args.batch, wall)}
    print(json.dumps(line), flush=True)


def workload_config(args, world):
    return {"workload": "BASELINE config 4 per-GPU shard: Text2Mel AR (210 frames) + SSRN, "
                        "%d synthetic %d-char utterances per GPU, LJ hyper-parameters" % (args.batch, args.nchars),
            "batch_per_gpu": args.batch, "global_batch": args.batch * world, "max_N": 180, "max_T": 210,
            "parallelism": "utterance-shard x%d + one NCCL gather of Z to rank 0 (chunked, overlapped with the SSRN)" % world,
            "l2": "flushed between timed steps (256 MiB write, untimed); per-step working set "
                  "(weights 210 MB + activations) also exceeds the 50 MB L2"}


# ------------------------------------------------------------------------------ CUDA arm
# Algorithmic work of the path (SURVEY.md 8a / 8d), per utterance
MAC_TEXTENC_PER_CHAR = 17104896            # TextEnc, per character position (N = 180 positions)
MAC_AUDIOENC_PER_FRAME = 4083712
MAC_AUDIODEC_PER_FRAME = 2707456
MAC_SSRN_PER_FRAME = 93655052
DECODE_WEIGHT_BYTES = (4101376 + 2719984) * 4          # AudioEnc + AudioDec parameters, fp32: read once per mel frame


def parity_sample(eng, params, L_row, Y_row, Z_row, P_row):
    """Oracle check of ONE utterance of the timed output (free running, all frames): asserts max-abs <= 1e-3 on mel and
    linear magnitudes up to the first near-tie of the argmax feedback (margin < 1e-4), identical windows there."""
    import numpy as np
    import torch
    from oracle import ref_torch as rt
    torch.set_num_threads(usable_cores())
    T = Y_row.shape[0]
    r = rt.synthesize(params, L_row[None], steps=T, literal=False, record=True)
    Yo, Po, mg = r["Y"].numpy()[0], r["p_hist"].numpy()[0], r["margin_hist"].numpy()[0]
    bad = np.nonzero(mg < 1e-4)[0]
    n = int(bad[0]) + 1 if bad.size else T
    same_p = bool(np.array_equal(P_row[:n], Po[:n]))
    dy = float(np.abs(Y_row[:n] - Yo[:n]).max())
    dz = None
    if n == T:
        dz = float(np.abs(Z_row - r["Z"].numpy()[0]).max())
    out = {"utterance": 0, "frames_checked": n, "windows_equal": same_p, "max_abs_mel": dy, "max_abs_mag": dz,
           "tolerance": 1e-3, "oracle": "oracle/ref_torch.synthesize (reference schedule)"}
    if not (same_p and dy <= 1e-3 and (dz is None or dz <= 1e-3)):
        raise AssertionError("bench parity check failed: %s" % json.dumps(out))
    return out


DUMP_BYTES = 64 << 20


def dump_outputs(out_dir, Y, Z, P):
    """What the last timed step returned, as float32 / float64 .npy files, over the global batch of all ranks (U = N * batch
    utterances in rank order): mel (U, T, n_mels), mag (U, 4T, 1+n_fft/2) and the attention window of every frame (U, T).
    When everything does not fit DUMP_BYTES, mag keeps a fixed, seeded sample of utterances; mag_rows.npy lists their
    indices into the global batch."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    mel = Y.float().cpu().numpy()
    win = P.cpu().numpy().astype(np.float64)
    per_utt = Z[0].numel() * 4
    room = DUMP_BYTES - mel.nbytes - win.nbytes
    rows = np.arange(Z.shape[0])
    if room < per_utt * Z.shape[0]:
        k = max(1, room // per_utt)
        rows = np.sort(np.random.default_rng(0).choice(Z.shape[0], size=k, replace=False))
        np.save(os.path.join(out_dir, "mag_rows.npy"), rows.astype(np.float64))
    np.save(os.path.join(out_dir, "mel.npy"), mel)
    np.save(os.path.join(out_dir, "mag.npy"), Z[torch.as_tensor(rows, device=Z.device)].float().cpu().numpy())
    np.save(os.path.join(out_dir, "attention_windows.npy"), win)


def run_b200(args, rank, local_rank, world):
    import numpy as np
    import torch
    import torch.distributed as dist
    from dc_tts_b200.engine import Engine
    from dc_tts_b200.hyperparams import Hyperparams as hp
    from dc_tts_b200.parallel import OverlappedGather
    from dc_tts_b200.params import init_params, synthetic_text

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    params = init_params(0, "perturbed")
    eng = Engine(local_rank)
    eng.load_params(params)
    eng.set_tensor_path(args.tensor_path)
    eng.set_option("decode_mode", args.decode_mode)
    B, T, F = args.batch, hp.max_T, 1 + hp.n_fft // 2
    eng.reserve(B)
    L_np = synthetic_text(B, args.nchars, seed=0, first_index=rank * B)
    L_host = torch.from_numpy(L_np).pin_memory()
    L_dev = L_host.to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    total = B * world
    # finished spectrograms: rank 0 receives every rank's Z; chunks leave while the SSRN of the next chunk runs
    n_chunks = args.gather_chunks if args.gather_chunks > 0 else (1 if world <= 4 else 2)
    og = OverlappedGather(total, (T * hp.r, F), torch.float32, dev, chunks=n_chunks) if world > 1 else None
    Zloc = torch.empty((B, T * hp.r, F), device=dev) if (world == 1 or rank != 0) else None
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def step(marks=None):
        Y, P, _, _ = eng.text2mel_generate(L_dev)
        if marks is not None:
            marks[0].record()
        if world == 1:
            eng.ssrn(Y, want_logits=False, out=Zloc)
            Z = Zloc
            if marks is not None:
                marks[1].record()
        else:
            og.begin()
            for c in og.chunks():
                view = og.local_view(c)
                out = view if view is not None else Zloc[c.lo:c.hi]
                eng.ssrn(Y[c.lo:c.hi], want_logits=False, out=out)
                og.send(c, out)
            if marks is not None:
                marks[1].record()
            Z = og.finish()
        return Y, Z, P

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        step()
    barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    launches0 = eng.launch_count()
    evs = [(ev(), ev(), ev(), ev()) for _ in range(args.steps)]
    barrier()
    for k in range(args.steps):
        flush.fill_(k & 0xff)                      # L2 flush, outside the per-step event pair
        evs[k][0].record()
        Y, Z, P = step(marks=(evs[k][1], evs[k][2]))
        evs[k][3].record()
    barrier()
    if args.dump_outputs:
        Yd, Pd = Y, P
        if world > 1:                              # rank 0 holds the gathered magnitudes: gather mel and windows too
            Yd = torch.empty((total,) + tuple(Y.shape[1:]), dtype=Y.dtype, device=dev)
            Pd = torch.empty((total,) + tuple(P.shape[1:]), dtype=P.dtype, device=dev)
            dist.all_gather_into_tensor(Yd, Y.contiguous())
            dist.all_gather_into_tensor(Pd, P.contiguous())
        if rank == 0:
            dump_outputs(args.dump_outputs, Yd, Z, Pd)
    ms = sum(e[0].elapsed_time(e[3]) for e in evs)
    ms_t2m = sum(e[0].elapsed_time(e[1]) for e in evs) / args.steps
    ms_ssrn = sum(e[1].elapsed_time(e[2]) for e in evs) / args.steps
    ms_tail = sum(e[2].elapsed_time(e[3]) for e in evs) / args.steps
    launches = eng.launch_count() - launches0
    clocks = sampler.stop() if rank == 0 else None
    t = torch.tensor([ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t.item())
    value = total * T * args.steps / (ms / 1e3)
    dstats = eng.decode_stats() if args.decode_mode == 1 else None

    # ---- e2e: public host-buffer API, H2D + D2H inside the timed region (per rank, max over ranks)
    Yh = torch.empty((B, T, hp.n_mels)).pin_memory()
    Zh = torch.empty((B, T * hp.r, F)).pin_memory()
    eng.synthesize_host(L_host, Yh, Zh)
    barrier()
    e2e_steps = max(1, min(args.steps, 5))
    t0 = time.perf_counter()
    for _ in range(e2e_steps):
        eng.synthesize_host(L_host, Yh, Zh)
    barrier()
    te = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(te, op=dist.ReduceOp.MAX)
    e2e_value = total * T * e2e_steps / float(te.item())

    # ---- BASELINE config 5 (SURVEY 8f-3): Text2Mel training step -- forward with dropout, losses, backward, clip, Adam -- at the
    # benchmark batch per GPU, data parallel over the launched ranks (NCCL all-reduce of the flat gradient arena); own handle
    # (a trained handle stops using the packed synthesis weights).  Not part of `value`.
    train = None
    if args.train_steps > 0:
        teng = Engine(local_rank)
        teng.load_params(init_params(0))
        teng.set_option("train_tc", args.train_tc)
        teng.train_init(B)
        mels = torch.from_numpy(np.random.default_rng(rank).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)).to(dev)
        grads = teng.train_grads()

        def tstep(i):
            o = teng.train_step(L_dev, mels, global_step=4000 + i, seed=i * world + rank, apply=(world == 1))
            if world > 1:
                dist.all_reduce(grads)
                grads.mul_(1.0 / world)
                teng.train_apply(4000 + i)
            return o
        for i in range(3):
            first = tstep(i)
        barrier()
        n0 = teng.launch_count()
        ta, tb = ev(), ev()
        ta.record()
        for i in range(args.train_steps):
            last = tstep(3 + i)
        tb.record()
        barrier()
        tt = torch.tensor([ta.elapsed_time(tb) / args.train_steps], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        tms = float(tt.item())
        tfl = 3 * 2 * B * (hp.max_N * MAC_TEXTENC_PER_CHAR + T * (MAC_AUDIOENC_PER_FRAME + MAC_AUDIODEC_PER_FRAME))   # fwd MACs x 2 x 3 GEMMs
        train = {"config": "BASELINE config 5: Text2Mel train step (fwd + bwd + clip + Adam), B=%d per GPU, N=180, T=210, dropout %.2f, "
                           "dp%d (all-reduce of %d gradients)" % (B, hp.dropout_rate, world, grads.numel()),
                 "ms_per_step": tms, "steps_per_sec": 1e3 / tms, "mel_frames_per_sec": world * B * T * 1e3 / tms, "steps": args.train_steps,
                 "achieved_tflops": world * tfl / (tms * 1e-3) / 1e12, "gpu_launches_per_step": (teng.launch_count() - n0) // args.train_steps,
                 "dtype": ("f32 tensors; forward / data-gradient / weight-gradient GEMMs as split-fp16 x3 on wgmma, fp32 accumulate"
                           if args.train_tc else "f32 (CUDA-core kernels)"),
                 "loss_first": first["loss"], "loss_last": last["loss"], "scaling": "weak"}
        teng.close()
        del teng, grads, mels
        torch.cuda.empty_cache()

    if rank == 0:
        peaks = measured_peaks()
        tensor = args.tensor_path != 0
        step_ms = ms / args.steps
        # ---- stage timings inside the timed step (rank 0): TextEnc is timed on its own, decode = generate - TextEnc
        for _ in range(2):
            eng.textenc(L_dev)
        a, b = ev(), ev()
        a.record()
        for _ in range(5):
            eng.textenc(L_dev)
        b.record(); torch.cuda.synchronize()
        ms_te = a.elapsed_time(b) / 5
        ms_dec = max(ms_t2m - ms_te, 1e-6)
        fl_te = 2.0 * B * hp.max_N * MAC_TEXTENC_PER_CHAR
        fl_dec = 2.0 * B * T * (MAC_AUDIOENC_PER_FRAME + MAC_AUDIODEC_PER_FRAME + 2 * hp.attention_win_size * hp.d)
        fl_ssrn = 2.0 * B * T * MAC_SSRN_PER_FRAME
        by_dec = float(T) * (DECODE_WEIGHT_BYTES + B * 4 * (hp.n_mels * 2 + 24 * 256 * 4))    # weights once per frame + rows in/out
        tf_peak = peaks["tf_sustained"] or peaks["tf"]
        stages = [
            {"stage": "TextEnc (wgmma blocks, once per batch)", "ms": ms_te, "share": ms_te / step_ms, "bound": "tensor",
             "algorithmic_flops": fl_te, "achieved_tflops": fl_te / ms_te / 1e9, "frac": fl_te / ms_te / 1e9 / tf_peak},
            {"stage": "decode: 210 frames of AudioEnc + Attention + AudioDec (%s)"
                      % ("ONE persistent cluster kernel" if args.decode_mode == 1 else "one CUDA graph per frame"),
             "ms": ms_dec, "us_per_frame": 1e3 * ms_dec / T, "share": ms_dec / step_ms, "bound": "hbm",
             "algorithmic_bytes": by_dec, "achieved_gbs": by_dec / ms_dec / 1e6, "frac": by_dec / ms_dec / 1e6 / peaks["hbm_gbs"],
             "useful_flops": fl_dec, "useful_tflops": fl_dec / ms_dec / 1e9,
             "note": "latency-bound recurrence: algorithmic bytes = the 27.3 MB of AudioEnc+AudioDec weights once per frame "
                     "(SURVEY 8d config 2); the receptive-field recompute after a window move (quirk Q1) is extra work, not "
                     "counted as useful",
             "window_moves": (None if dstats is None else {"cluster_frames_with_recompute": dstats[0],
                                                           "utterance_frames_recomputed": dstats[1], "clusters": dstats[2],
                                                           "of_utterance_frames": B * T})},
            {"stage": "SSRN (wgmma blocks)", "ms": ms_ssrn, "share": ms_ssrn / step_ms, "bound": "tensor",
             "algorithmic_flops": fl_ssrn, "achieved_tflops": fl_ssrn / ms_ssrn / 1e9, "frac": fl_ssrn / ms_ssrn / 1e9 / tf_peak,
             "tensor_pipe_frac_executed": 3 * fl_ssrn / ms_ssrn / 1e9 / tf_peak},
            {"stage": "gather tail (exposed part of the NCCL gather)", "ms": ms_tail, "share": ms_tail / step_ms},
        ]
        # ---- roofline of the dominant kernel of the timed step
        rows = B * T * hp.r
        kms = eng.bench_block("SSRN/HC_11", B, T * hp.r, iters=5, warmup=2)
        flops = 2.0 * rows * 3 * 1024 * 2048
        k_ms = kms[1] if tensor else kms[0]          # tensor path: [fp32->planes, fused block]; fp32 path: [GEMM, LN]
        ach = flops / (k_ms * 1e-3) / 1e12
        hc11 = {"kernel": ("conv_ln_tc_kernel: SSRN/HC_11 fused hc block on wgmma (M=%d, K=3x1024, N=2048, 3 fp16 MMA "
                           "passes per k-step)" if tensor else "conv_gemm_tiled: SSRN/HC_11 conv-GEMM on fp32 cores (M=%d, K=3x1024, N=2048)") % rows,
                "bound": "tensor", "achieved": ach, "peak": peaks["tf"], "unit": "TFLOP/s", "frac": ach / peaks["tf"],
                "algorithmic_bytes": int(rows * 1024 * 4 * 2 + 2 * 3 * 1024 * 2048 * 2),
                "peak_source": peaks["src"] + " bf16/fp16 dense (burst)",
                "kernel_ms": k_ms, "other_kernels_of_block_ms": [m for i, m in enumerate(kms) if m != k_ms],
                "share_of_step": 2 * k_ms / step_ms,
                "tensor_pipe_flops_executed_tflops": (3 * ach if tensor else 0.0),
                "note": "achieved = ALGORITHMIC FLOPs 2*M*K*N / CUDA-event time of that launch; the split-fp16 "
                        "scheme needed for the 1e-3 parity budget executes 3x that on the tensor pipe, so frac <= 1/3"}
        if args.decode_mode == 1 and ms_dec >= ms_ssrn:
            roof = {"kernel": "decode_cluster_kernel: the whole AR loop (210 frames x 24 conv blocks + attention) in one launch, "
                              "%d clusters x 16 CTAs" % (dstats[2] if dstats else 0),
                    "bound": "hbm", "achieved": by_dec / ms_dec / 1e6, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                    "frac": by_dec / ms_dec / 1e6 / peaks["hbm_gbs"],
                    "algorithmic_bytes": int(by_dec), "peak_source": peaks["src"] + " HBM copy bandwidth", "kernel_ms": ms_dec,
                    "share_of_step": ms_dec / step_ms,
                    "note": "dominant kernel of the timed step; a dependent-latency chain (24 blocks x 210 frames), not a streaming "
                            "kernel: its weights stay in L2 (27 MB < 50 MB), so DRAM traffic per launch is far below the "
                            "algorithmic bytes and the HBM roofline fraction mostly measures how short the chain is"}
        else:
            roof = hc11
        # ---- single-utterance latency (BASELINE config 2 + SSRN): RTF target >= 200x
        L1 = L_dev[:1].contiguous()
        for _ in range(2):
            Y1, _, _, _ = eng.text2mel_generate(L1); eng.ssrn(Y1, want_logits=False)
        torch.cuda.synchronize()
        a, b, c = ev(), ev(), ev()
        a.record(); Y1, _, _, _ = eng.text2mel_generate(L1); b.record(); eng.ssrn(Y1, want_logits=False); c.record()
        torch.cuda.synchronize()
        t2m_ms, ssrn1_ms = a.elapsed_time(b), b.elapsed_time(c)
        audio_s = T * hp.r * hp.hop_length / float(hp.sr)
        by1 = float(T) * DECODE_WEIGHT_BYTES
        single = {"config": "BASELINE config 2 (+ SSRN): B=1, 210 frames", "text2mel_ms": t2m_ms, "ssrn_ms": ssrn1_ms,
                  "us_per_frame": 1e3 * t2m_ms / T, "rtf_x_realtime": audio_s / ((t2m_ms + ssrn1_ms) / 1e3),
                  "roofline": {"bound": "hbm", "algorithmic_bytes": by1, "achieved_gbs": by1 / t2m_ms / 1e6,
                               "frac": by1 / t2m_ms / 1e6 / peaks["hbm_gbs"]}}
        ssrn3 = {"config": "BASELINE config 3: SSRN B=%d, T=210" % B, "ms": ms_ssrn, "achieved_tflops": fl_ssrn / ms_ssrn / 1e9,
                 "frac_of_tensor_peak": fl_ssrn / ms_ssrn / 1e9 / tf_peak, "peak": tf_peak,
                 "peak_source": peaks["src"] + " bf16/fp16 dense (sustained: timed inside the step)"}
        # ---- parity of the timed output against the oracle (one utterance, all frames)
        parity = None
        if args.parity_check and world == 1:
            parity = parity_sample(eng, params, L_np[0], Y[0].cpu().numpy(), Z[0].cpu().numpy(), P[0].cpu().numpy())
        cpu = cpu_baseline_block(args) if (args.cpu_passes > 0 and world == 1) else None   # rank 0, N = 1 only
        # ---- next row (SURVEY 8f): Griffin-Lim vocoder on this rank's finished spectrograms (not part of `value`)
        voc = None
        if world == 1:
            Zv = Z
            eng.spectrogram2wav(Zv); torch.cuda.synchronize()
            t0 = time.perf_counter(); wv, _ = eng.spectrogram2wav(Zv); torch.cuda.synchronize(); dtv = time.perf_counter() - t0
            hbm = 50 * (2 * 8 + 4 + 2 * 4 * 1102 / 1025.0) * B * T * hp.r * F + 51 * 2 * 4 * B * wv.shape[1]   # X r/w, S, frames r/w, wav r/w
            voc = {"what": "spectrogram2wav (Griffin-Lim, %d iterations, n_fft 2048) for %d utterances" % (hp.n_iter, B),
                   "ms": dtv * 1e3, "x_realtime": B * wv.shape[1] / float(hp.sr) / dtv,
                   "hbm_bytes_algorithmic": int(hbm), "hbm_frac_of_measured_peak": hbm / dtv / 1e9 / peaks["hbm_gbs"]}
        line = {"metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps,
                "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "f32 (decode: fp32 FMA; TextEnc/SSRN: fp16x2 split operands on wgmma, fp32 accumulate)" if args.tensor_path else "f32", "data": "synthetic",
                "config": workload_config(args, world),
                "clocks": clocks, "gpu_launches": launches,
                "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": int(L_host.numel() * 4),
                        "d2h_bytes_per_step": int((Yh.numel() + Zh.numel()) * 4), "steps": e2e_steps,
                        "api": "dctts_synthesize_host (pinned host buffers)"},
                "roofline": roof, "roofline_tensor_kernel": hc11, "stages": stages,
                "single_utterance": single, "ssrn_config3": ssrn3}
        if parity:
            line["parity_check"] = parity
        if voc:
            line["next_row_vocoder"] = voc
        if cpu:
            line["cpu_baseline"] = cpu
        if train:
            line["train_config5"] = train
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--batch", type=int, default=32, help="utterances per GPU")
    ap.add_argument("--nchars", type=int, default=100)
    ap.add_argument("--cpu-passes", type=int, default=6, help="full-graph passes (at the benchmark batch) of the CPU baseline sample (0 = skip)")
    ap.add_argument("--decode-mode", type=int, default=1, choices=[0, 1], help="1 = persistent cluster decode kernel (default), 0 = one CUDA graph per frame")
    ap.add_argument("--gather-chunks", type=int, default=0, help="N > 1: SSRN / gather chunks per rank (transfer of a chunk runs under the next chunk's SSRN); "
                    "0 = auto: 1 up to 4 GPUs, 2 beyond (every extra chunk leaves partly filled waves in the SSRN, while rank 0's ingest "
                    "grows with N)")
    ap.add_argument("--no-parity-check", dest="parity_check", action="store_false", help="skip the oracle check of the timed output")
    ap.add_argument("--tensor-path", type=int, default=1, choices=[0, 1], help="1 = tensor-core (wgmma) blocks (default), 0 = fp32 CUDA-core kernels only")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="write what the last timed step computed (mel, mag, "
                    "attention windows) as .npy files under DIR")
    ap.add_argument("--train-steps", type=int, default=5, help="timed steps of the BASELINE config 5 training step reported as train_config5 (0 = skip)")
    ap.add_argument("--train-tc", type=int, default=7, help="training GEMMs on the tensor cores, bit mask (1 forward, 2 data gradient, 4 weight gradient); 0 = fp32 CUDA cores")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world == 1 and args.gpus > 1 and args.impl == "b200":
        # convenience: re-launch under torchrun, one rank per GPU
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus),
               "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 400)] + sys.argv
        sys.exit(subprocess.call(cmd))
    if args.impl == "reference":
        run_reference(args, rank, world)
    else:
        run_b200(args, rank, local_rank, world)


if __name__ == "__main__":
    main()
