"""Engine: one libdctts_b200 handle bound to one GPU, driven with torch device tensors.

torch is used here for device memory and streams only; every computation goes through
the C-ABI (include/dctts.h).  This object plays the role of the reference's
`tf.Session` + restored variables (/root/reference/synthesize.py:28-41).
"""
import ctypes as C
import warnings
import weakref

import numpy as np
import torch

from . import _lib
from .hyperparams import Hyperparams as hp
from .params import check_params


class DcttsError(RuntimeError):
    pass


def _ptr(t):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def _require_tensors(who, want):
    """Each (tensor, shape, dtype) of `want` is a contiguous CUDA tensor of that shape and dtype, else DcttsError."""
    for t, shape, dt in want:
        if tuple(t.shape) != shape or t.dtype != dt or not t.is_cuda or not t.is_contiguous():
            raise DcttsError("%s: expected a contiguous CUDA %s tensor of shape %s, got %s %s" %
                             (who, dt, shape, t.dtype, tuple(t.shape)))


def _host(x):
    """A list, numpy array or tensor on any device as a host numpy array."""
    return np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x)


def _host_ints(who, x, B, name, lo=-2 ** 31, hi=2 ** 31 - 1):
    """`x` (a list, numpy array or tensor on any device) as a host int64 vector of B values, each in [lo, hi]; else
    DcttsError "<who>: <n> <name>s for <B> utterances" or "<who>: utterance <b> has <name> <v> outside [lo, hi]".  The
    default range is int32's, the type every entry point takes."""
    v = _host(x).astype(np.int64).reshape(-1)
    if v.shape[0] != B:
        raise DcttsError("%s: %d %ss for %d utterances" % (who, v.shape[0], name, B))
    bad = np.flatnonzero((v < lo) | (v > hi))
    if bad.size:
        raise DcttsError("%s: utterance %d has %s %d outside [%d, %d]" % (who, bad[0], name, v[bad[0]], lo, hi))
    return v


class Engine:
    def __init__(self, device=0, hparams=hp):
        self._lib = _lib.load()
        if not torch.cuda.is_available():
            raise DcttsError("dc_tts_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        self.hp = hparams
        self.F = 1 + hparams.n_fft // 2
        st = _lib.HParams(len(hparams.vocab), hparams.e, hparams.d, hparams.c, hparams.n_mels,
                          hparams.n_fft, hparams.max_N, hparams.max_T, hparams.attention_win_size, hparams.r)
        h = _lib.Handle()
        torch.cuda.init()
        with torch.cuda.device(self.device):
            torch.zeros(1, device=self.device)          # make sure the primary context exists
            rc = self._lib.dctts_create(C.byref(st), device, C.byref(h))
        if rc != 0:
            raise DcttsError("dctts_create: " + self._lib.dctts_last_error(None).decode())
        self._h = h
        self.params_loaded = False
        self._streams = weakref.WeakSet()   # open VocoderStreams and SynthesisStreams: closed before the handle they hold

    # ------------------------------------------------------------------ plumbing
    def close(self):
        for vs in list(getattr(self, "_streams", ())):
            vs._free()
        if getattr(self, "_h", None):
            self._lib.dctts_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise DcttsError("%s: %s" % (what, self._lib.dctts_last_error(self._h).decode()))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _f32(self, x):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        return x.to(device=self.device, dtype=torch.float32).contiguous()

    def _i32(self, x):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.int32))
        return torch.as_tensor(x).to(device=self.device, dtype=torch.int32).contiguous()

    def _empty(self, *shape, dtype=torch.float32):
        return torch.empty(shape, device=self.device, dtype=dtype)

    # ------------------------------------------------------------------ parameters
    def stage_params(self, params):
        """Stage some variables (e.g. one of the two checkpoints of synthesize.py:31-41); commit_params() uploads."""
        for name, arr in params.items():
            a = np.ascontiguousarray(arr, dtype=np.float32)
            shape = (C.c_int64 * a.ndim)(*a.shape)
            self._check(self._lib.dctts_set_param(self._h, name.encode(), a.ctypes.data_as(C.c_void_p),
                                                   shape, a.ndim), "dctts_set_param(%s)" % name)

    def commit_params(self):
        """Fails (library error) when a variable of the path is missing or mis-shaped."""
        self._check(self._lib.dctts_commit_params(self._h), "dctts_commit_params")
        self.params_loaded = True
        return int(self._lib.dctts_num_params(self._h))

    def load_params(self, params):
        """Stage every variable (TF names, SURVEY.md App. C) and commit them to the device."""
        check_params(params)
        self.stage_params(params)
        return self.commit_params()

    def restore(self, text2mel_dir, ssrn_dir=None):
        """synthesize.py:31-41: the latest Text2Mel checkpoint of `<logdir>-1` and SSRN checkpoint of `<logdir>-2`
        (TF tensor bundles, read without TensorFlow by dc_tts_b200/checkpoint.py)."""
        from .checkpoint import Saver, latest_checkpoint
        Saver(var_list=["Text2Mel"]).restore(self, latest_checkpoint(text2mel_dir))
        Saver(var_list=["SSRN", "gs"]).restore(self, latest_checkpoint(ssrn_dir if ssrn_dir is not None else text2mel_dir))
        return self.commit_params()

    def set_tensor_path(self, mode):
        self._check(self._lib.dctts_set_tensor_path(self._h, int(mode)), "dctts_set_tensor_path")

    def set_option(self, name, value):
        """Kernel-variant switch (include/dctts.h: dctts_set_option), e.g. ("decode_mode", 0) for the graph-per-frame loop."""
        self._check(self._lib.dctts_set_option(self._h, name.encode(), int(value)), "dctts_set_option(%s)" % name)

    def get_option(self, name):
        v = C.c_int32(0)
        self._check(self._lib.dctts_get_option(self._h, name.encode(), C.byref(v)), "dctts_get_option(%s)" % name)
        return int(v.value)

    def decode_stats(self):
        """(frames with a receptive-field recompute summed over clusters, utterance-frames recomputed, clusters)."""
        a, b, c = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._check(self._lib.dctts_decode_stats(self._h, C.byref(a), C.byref(b), C.byref(c)), "dctts_decode_stats")
        return int(a.value), int(b.value), int(c.value)

    def decode_profile(self):
        """Lap timers (SM cycles) of the last persistent decode run with option decode_prof = 1; see include/dctts.h."""
        names = ["start", "stream_wait", "gemv", "release", "gather", "cluster_barrier", "layernorm", "mix", "attention",
                 "re_attention", "re_weights", "re_table", "re_stage", "re_drain", "re_refill", "re_layernorm", "re_barriers",
                 "frame", "wg_a_wait", "wg_mma", "wg_epilogue", "prefetch"]
        v = (C.c_int64 * len(names))()
        self._check(self._lib.dctts_decode_profile(self._h, v, len(names)), "dctts_decode_profile")
        return dict(zip(names, [int(x) for x in v]))

    def reserve(self, batch):
        self._check(self._lib.dctts_reserve(self._h, int(batch)), "dctts_reserve")

    def reserve_frames(self, batch, frames):
        """Grow the full-sequence chains' workspace to `batch` utterances of `frames` mel frames, above max_T too
        (include/dctts.h: dctts_reserve_frames); returns the bytes those buffers hold afterwards."""
        n = C.c_int64(0)
        self._check(self._lib.dctts_reserve_frames(self._h, int(batch), int(frames), C.byref(n)), "dctts_reserve_frames")
        return n.value

    def join_rows(self, Y, lengths, piece_text, piece_pause, K, silence=1e-8):
        """The long-form join (include/dctts.h: dctts_join_rows): Y (P, T, n_mels) decoded pieces, lengths (P,) int32 CUDA
        tensor (as text2mel_generate_until returns it), piece_text / piece_pause (P,) host integers.  Returns (out
        (K, T_out, n_mels), out_len (K,) int32 CUDA tensor), T_out the longest text at full-length pieces; one launch and
        no synchronisation."""
        Y = self._f32(Y)
        P, T, Cm = Y.shape
        n = self._i32(lengths).reshape(-1)
        if Cm != self.hp.n_mels or n.shape[0] != P:
            raise DcttsError("join_rows: Y (P, T, %d) with P lengths, got Y %s and %d lengths"
                             % (self.hp.n_mels, tuple(Y.shape), n.shape[0]))
        text = np.ascontiguousarray(_host_ints("join_rows", piece_text, P, "piece text"), np.int32)
        pause = np.ascontiguousarray(_host_ints("join_rows", piece_pause, P, "piece pause"), np.int32)
        K = int(K)
        if K < 1 or P < 1 or text.min() < 0 or text.max() >= K:
            raise DcttsError("join_rows: need P >= 1 pieces whose texts lie in [0, K = %d)" % K)
        T_out = int(max(np.bincount(text, weights=T + pause.astype(np.int64), minlength=K)))
        out = self._empty(K, T_out, Cm)
        out_len = self._empty(K, dtype=torch.int32)
        self._check(self._lib.dctts_join_rows(self._h, _ptr(Y), P, T, _ptr(n), text.ctypes.data_as(C.c_void_p),
                                              pause.ctypes.data_as(C.c_void_p), K, float(silence), T_out, _ptr(out),
                                              _ptr(out_len), self._stream()), "dctts_join_rows")
        return out, out_len

    def bench_block(self, scope, B, L, iters=5, warmup=2):
        """Mean device milliseconds of each kernel of one block (roofline leg of bench.py)."""
        ms = (C.c_float * 8)()
        n = C.c_int32(0)
        self._check(self._lib.dctts_bench_block(self._h, scope.encode(), B, L, iters, warmup, ms, C.byref(n),
                                                self._stream()), "dctts_bench_block")
        return [float(ms[i]) for i in range(n.value)]

    def conv_gemm(self, impl, mode, X, K, Wd, N, shifts, out, bias=None, accumulate=0):
        """Test aid (include/dctts.h: dctts_conv_gemm): one conv-GEMM of the training step, in place on `out`.
        impl 0 = fp32 CUDA-core kernels, 1 = wgmma.  Every tensor is a CUDA float32 view with unit stride in its last dim;
        the row pitches are the views' strides.  X (B, L, >= K).  Mode 0: Wd (ntaps, K, >= N) = W, out (B, L, ldo), bias.
        Mode 1: Wd (B, L, >= N) = dY, out (ntaps, K, >= N) += the weight gradient."""
        ts = [X, Wd, out] + ([bias] if bias is not None else [])
        if not all(t.is_cuda and t.dtype == torch.float32 and t.stride(-1) == 1 for t in ts):
            raise DcttsError("conv_gemm: CUDA float32 tensors with a unit inner stride expected")
        B, L = X.shape[0], X.shape[1]
        rows_ok = X.stride(0) == L * X.stride(1) and (mode == 1 or out.stride(0) == L * out.stride(1))
        taps_ok = (Wd.stride(0) == K * Wd.stride(1)) if mode == 0 else (out.stride(0) == K * out.stride(1))
        dy_ok = mode == 0 or (Wd.shape[0] == B and Wd.shape[1] == L and Wd.stride(0) == L * Wd.stride(1))
        if not (rows_ok and taps_ok and dy_ok):
            raise DcttsError("conv_gemm: rows or taps of a tensor are not evenly pitched")
        sh = (C.c_int32 * len(shifts))(*[int(s) for s in shifts])
        self._check(self._lib.dctts_conv_gemm(self._h, int(impl), int(mode), _ptr(X), X.stride(1), B, L, int(K), _ptr(Wd),
                                              Wd.stride(1), int(N), len(shifts), sh, _ptr(bias), int(accumulate), _ptr(out),
                                              out.stride(1), self._stream()), "dctts_conv_gemm")
        return out

    @staticmethod
    def _pitched(who, ts, rows):
        """Each tensor of `ts` is a CUDA float32 view of `rows` rows with a unit inner stride, its rows evenly pitched (the
        pitch is the row stride); returns the pitches."""
        if not all(t.is_cuda and t.dtype == torch.float32 and t.stride(-1) == 1 for t in ts):
            raise DcttsError("%s: CUDA float32 tensors with a unit inner stride expected" % who)
        pitches = []
        for t in ts:
            lead = t.shape[:-1]
            n = 1
            for s in lead:
                n *= s
            ld = t.stride(-2) if t.dim() >= 2 else t.shape[-1]
            even = all(t.stride(i) == t.stride(i + 1) * t.shape[i + 1] for i in range(t.dim() - 2))
            if n != rows or not even:
                raise DcttsError("%s: rows of a tensor are not evenly pitched, or not %d of them" % (who, rows))
            pitches.append(ld)
        return pitches

    def block_bwd(self, mode, act, C, pre, gout, ln, dy, dparams, X=None, gin=None, dropout_rate=0.0, layer=0, seed=0):
        """Test aid (include/dctts.h: dctts_block_bwd): the dropout / activation / highway / LayerNorm backward of one block,
        one launch.  pre, dy (rows, >= nconv); gout (rows, >= C); X, gin (rows, >= C) for mode 1 (highway); ln (4, C) =
        g1 | b1 | g2 | b2 contiguous; dparams (4 C + nconv) contiguous, added onto.  Leading dims are flattened into rows;
        the pitches are the views' row strides."""
        nconv = 2 * C if mode == 1 else C
        if mode == 1 and (X is None or gin is None):
            raise DcttsError("block_bwd: a highway block (mode 1) needs X and gin")
        rows = 1
        for s in pre.shape[:-1]:
            rows *= s
        ts = [pre, gout, dy] + ([X, gin] if mode == 1 else [])
        if any(t.shape[-1] < w for t, w in zip(ts, (nconv, C, nconv, C, C))):
            raise DcttsError("block_bwd: pre and dy need %d columns, gout, X and gin %d" % (nconv, C))
        lds = self._pitched("block_bwd", ts, rows)
        if gout.stride(-2) != lds[1] or (mode == 1 and gin.stride(-2) != lds[1]):
            raise DcttsError("block_bwd: gout and gin share one pitch")
        if dy.stride(-2) != lds[0]:
            raise DcttsError("block_bwd: pre and dy share one pitch")
        _require_tensors("block_bwd", [(ln, (4, C), torch.float32), (dparams, (4 * C + nconv,), torch.float32)])
        self._check(self._lib.dctts_block_bwd(self._h, int(mode), int(act), rows, int(C), _ptr(pre), lds[0], _ptr(gout), lds[1],
                                              _ptr(X), lds[3] if mode == 1 else 0, _ptr(ln), float(dropout_rate), int(layer),
                                              int(seed) & 0xffffffff, _ptr(dy), _ptr(gin), _ptr(dparams), self._stream()),
                    "dctts_block_bwd")
        return dy

    def block_fwd(self, mode, act, C, pre, ln, out, X=None, dropout_rate=0.0, layer=0, seed=0):
        """Test aid (include/dctts.h: dctts_block_fwd): the training forward's LayerNorm / activation / highway / dropout
        epilogue of one block, one launch, into `out` (rows, >= C).  pre (rows, >= nconv); X (rows, >= C) for mode 1; ln (4, C)
        = g1 | b1 | g2 | b2 contiguous.  Leading dims are flattened into rows; the pitches are the views' row strides."""
        nconv = 2 * C if mode == 1 else C
        if mode == 1 and X is None:
            raise DcttsError("block_fwd: a highway block (mode 1) needs X")
        rows = 1
        for s in pre.shape[:-1]:
            rows *= s
        ts = [pre, out] + ([X] if mode == 1 else [])
        if any(t.shape[-1] < w for t, w in zip(ts, (nconv, C, C))):
            raise DcttsError("block_fwd: pre needs %d columns, out and X %d" % (nconv, C))
        lds = self._pitched("block_fwd", ts, rows)
        _require_tensors("block_fwd", [(ln, (4, C), torch.float32)])
        self._check(self._lib.dctts_block_fwd(self._h, int(mode), int(act), rows, int(C), _ptr(pre), lds[0], _ptr(X),
                                              lds[2] if mode == 1 else 0, _ptr(ln), float(dropout_rate), int(layer),
                                              int(seed) & 0xffffffff, _ptr(out), lds[1], self._stream()), "dctts_block_fwd")
        return out

    def attn_bwd(self, gR, Q, KV, align, gts, n_lim, t_lim, gQ, gKV, sums):
        """Test aid (include/dctts.h: dctts_attn_bwd): the attention backward of the Text2Mel step.  gR (B, T, 2d), Q (B, T, d),
        KV (B, N, 2d), align (B, N, T), gQ (B, T, d), gKV (B, N, 2d) contiguous; gts (>= n_lim, ld_gts) with a unit inner
        stride, its row stride the table's; sums (3,) float64, sums[2] added onto."""
        B, T, N, d = align.shape[0], align.shape[2], align.shape[1], self.hp.d
        f32 = torch.float32
        _require_tensors("attn_bwd", [(gR, (B, T, 2 * d), f32), (Q, (B, T, d), f32), (KV, (B, N, 2 * d), f32),
                                      (align, (B, N, T), f32), (gQ, (B, T, d), f32), (gKV, (B, N, 2 * d), f32),
                                      (sums, (3,), torch.float64)])
        if gts.dim() != 2 or gts.shape[0] < n_lim or gts.shape[1] < t_lim:
            raise DcttsError("attn_bwd: gts must be 2-D with at least n_lim = %d rows and t_lim = %d columns, got %s"
                             % (n_lim, t_lim, tuple(gts.shape)))
        ld_gts = self._pitched("attn_bwd", [gts], gts.shape[0])[0]
        self._check(self._lib.dctts_attn_bwd(self._h, _ptr(gR), _ptr(Q), _ptr(KV), _ptr(align), _ptr(gts), ld_gts, B, T, N,
                                             int(n_lim), int(t_lim), _ptr(gQ), _ptr(gKV), _ptr(sums), self._stream()),
                    "dctts_attn_bwd")
        return gQ, gKV

    def train_loss(self, logits, target, dlogits, sums, Y=None):
        """Test aid (include/dctts.h: dctts_train_loss): L1 + BCE on sigmoid(logits) against target, and the logits'
        gradient.  logits, dlogits (rows, >= C) views with a unit inner stride (the pitches are their row strides); target
        and Y (rows, C) contiguous; sums (2,) float64, added onto."""
        rows, C = target.shape
        if logits.shape[-1] < C or dlogits.shape[-1] < C:
            raise DcttsError("train_loss: logits and dlogits need %d columns" % C)
        ldl, ldg = self._pitched("train_loss", [logits, dlogits], rows)
        want = [(target, (rows, C), torch.float32), (sums, (2,), torch.float64)] + ([(Y, (rows, C), torch.float32)] if Y is not None else [])
        _require_tensors("train_loss", want)
        self._check(self._lib.dctts_train_loss(self._h, _ptr(logits), ldl, _ptr(target), rows, C, _ptr(dlogits), ldg, _ptr(Y),
                                               _ptr(sums), self._stream()), "dctts_train_loss")
        return dlogits

    def launch_count(self):
        return int(self._lib.dctts_launch_count(self._h))

    # ------------------------------------------------------------------ building blocks
    def embed(self, scope, ids):
        ids = self._i32(ids)
        B, N = ids.shape
        out = self._empty(B, N, self.hp.e)
        self._check(self._lib.dctts_embed(self._h, scope.encode(), _ptr(ids), B, N, _ptr(out), self._stream()), "dctts_embed")
        return out

    def normalize(self, scope, x):
        x = self._f32(x)
        Cc = x.shape[-1]
        out = torch.empty_like(x)
        self._check(self._lib.dctts_normalize(self._h, scope.encode(), _ptr(x), x.numel() // Cc, Cc, _ptr(out),
                                              self._stream()), "dctts_normalize")
        return out

    def conv1d(self, scope, x, filters, rate=1, causal=False, act=0):
        x = self._f32(x)
        B, L, _ = x.shape
        out = self._empty(B, L, filters)
        self._check(self._lib.dctts_conv1d(self._h, scope.encode(), _ptr(x), B, L, rate, int(causal), act,
                                           _ptr(out), self._stream()), "dctts_conv1d")
        return out

    def hc(self, scope, x, rate=1, causal=False):
        x = self._f32(x)
        B, L, _ = x.shape
        out = torch.empty_like(x)
        self._check(self._lib.dctts_hc(self._h, scope.encode(), _ptr(x), B, L, rate, int(causal), _ptr(out),
                                       self._stream()), "dctts_hc")
        return out

    def conv1d_transpose(self, scope, x):
        x = self._f32(x)
        B, L, Cc = x.shape
        out = self._empty(B, 2 * L, Cc)
        self._check(self._lib.dctts_conv1d_transpose(self._h, scope.encode(), _ptr(x), B, L, _ptr(out),
                                                     self._stream()), "dctts_conv1d_transpose")
        return out

    # ------------------------------------------------------------------ networks
    def textenc(self, L):
        L = self._i32(L)
        B, N = L.shape
        if N != self.hp.max_N:
            raise DcttsError("TextEnc: text must be padded to max_N=%d (reference networks.py:145)" % self.hp.max_N)
        K, V = self._empty(B, N, self.hp.d), self._empty(B, N, self.hp.d)
        self._check(self._lib.dctts_textenc(self._h, _ptr(L), B, _ptr(K), _ptr(V), self._stream()), "dctts_textenc")
        return K, V

    def audioenc(self, S):
        S = self._f32(S)
        B, T, _ = S.shape
        Q = self._empty(B, T, self.hp.d)
        self._check(self._lib.dctts_audioenc(self._h, _ptr(S), B, T, _ptr(Q), self._stream()), "dctts_audioenc")
        return Q

    def attention(self, Q, K, V, monotonic=False, prev_max_attentions=None):
        Q, K, V = self._f32(Q), self._f32(K), self._f32(V)
        B, T, d = Q.shape
        N = K.shape[1]
        pma = self._i32(prev_max_attentions) if monotonic else None
        R = self._empty(B, T, 2 * d)
        A = self._empty(B, N, T)
        M = self._empty(B, T, dtype=torch.int64)
        self._check(self._lib.dctts_attention(self._h, _ptr(Q), _ptr(K), _ptr(V), B, T, N, int(bool(monotonic)),
                                              _ptr(pma), _ptr(R), _ptr(A), _ptr(M), self._stream()), "dctts_attention")
        return R, A, M

    def audiodec(self, R):
        R = self._f32(R)
        B, T, _ = R.shape
        logits, Y = self._empty(B, T, self.hp.n_mels), self._empty(B, T, self.hp.n_mels)
        self._check(self._lib.dctts_audiodec(self._h, _ptr(R), B, T, _ptr(logits), _ptr(Y), self._stream()), "dctts_audiodec")
        return logits, Y

    def ssrn(self, Y, want_logits=True, out=None, lengths=None):
        """`out`: optional preallocated contiguous (B, 4T, F) float32 CUDA tensor (e.g. a slice of a gather buffer).
        T may exceed max_T (long-form synthesis): the workspace grows to B x T frames first (reserve_frames).
        `lengths`: optional (B,) mel frames per utterance, 1 <= lengths[b] <= T (include/dctts.h: dctts_ssrn_ragged):
        rows < 4 lengths[b] of Z and the logits are what this call gives for Y[b:b+1, :lengths[b]] alone, bit for bit, rows
        past them are 0, and Y rows >= lengths[b] are never read.  The range is checked on the host (one small copy)."""
        Y = self._f32(Y)
        B, T, _ = Y.shape
        if out is not None:
            if tuple(out.shape) != (B, T * self.hp.r, self.F) or out.dtype != torch.float32 or not out.is_contiguous() \
                    or out.device != self.device:
                raise DcttsError("ssrn: `out` must be a contiguous float32 (B, 4T, F) tensor on this engine's device")
        n = None
        if lengths is not None:
            n = self._i32(lengths).reshape(-1)
            _host_ints("ssrn", n, B, "length", 1, T)
        if T > self.hp.max_T:               # grow the workspace first: a size it cannot take is refused before any output
            self.reserve_frames(B, T)
        Z = out if out is not None else self._empty(B, T * self.hp.r, self.F)
        logits = self._empty(B, T * self.hp.r, self.F) if want_logits else None
        if n is None:
            self._check(self._lib.dctts_ssrn(self._h, _ptr(Y), B, T, _ptr(logits), _ptr(Z), self._stream()), "dctts_ssrn")
        else:
            self._check(self._lib.dctts_ssrn_ragged(self._h, _ptr(Y), B, T, _ptr(n), _ptr(logits), _ptr(Z), self._stream()),
                        "dctts_ssrn_ragged")
        return logits, Z

    # ------------------------------------------------------------------ graph level
    def text2mel_forward(self, L, mels, prev_max_attentions, want_alignments=True):
        L, mels, pma = self._i32(L), self._f32(mels), self._i32(prev_max_attentions)
        B = L.shape[0]
        if L.shape[1] != self.hp.max_N or mels.shape[1] != self.hp.max_T:
            raise DcttsError("synthesize graph needs N == max_N and T == max_T (reference networks.py:145)")
        Y = self._empty(B, self.hp.max_T, self.hp.n_mels)
        M = self._empty(B, self.hp.max_T, dtype=torch.int64)
        A = self._empty(B, self.hp.max_N, self.hp.max_T) if want_alignments else None
        self._check(self._lib.dctts_text2mel_forward(self._h, _ptr(L), _ptr(mels), _ptr(pma), B, _ptr(Y), _ptr(M),
                                                     _ptr(A), self._stream()), "dctts_text2mel_forward")
        return Y, M, A

    def text2mel_generate(self, L, steps=0, want_final_attention=False):
        L = self._i32(L)
        B = L.shape[0]
        Y = self._empty(B, self.hp.max_T, self.hp.n_mels)
        P = self._empty(B, self.hp.max_T, dtype=torch.int32)
        M = self._empty(B, self.hp.max_T, dtype=torch.int64) if want_final_attention else None
        A = self._empty(B, self.hp.max_N, self.hp.max_T) if want_final_attention else None
        self._check(self._lib.dctts_text2mel_generate(self._h, _ptr(L), B, int(steps), _ptr(Y), _ptr(P), _ptr(M),
                                                      _ptr(A), self._stream()), "dctts_text2mel_generate")
        self._decode_order = np.arange(B)
        return Y, P, M, A

    def text2mel_generate_until(self, L, stop_pos=None, tail=0, steps=0):
        """text2mel_generate with an end for each utterance (include/dctts.h: dctts_text2mel_generate_until): utterance b
        ends `tail` frames after the first frame whose attention argmax reaches stop_pos[b] (< 0: never).  stop_pos=None:
        the EOS positions of L (data_load.eos_positions).  Returns (Y, P, lengths): Y rows >= lengths[b] are 0, P rows
        >= lengths[b] are -1, and the rows below are those of text2mel_generate, bit for bit; lengths is an int32 CUDA
        tensor.  The utterances are decoded in the order of their stop positions, so that the utterances sharing a decode
        cluster end at similar frames; the outputs are in the caller's order."""
        from .data_load import eos_positions
        if tail < 0:
            raise DcttsError("text2mel_generate_until: tail must be >= 0")
        L = self._i32(L)
        B = L.shape[0]
        sp = eos_positions(L.cpu().numpy()) if stop_pos is None else \
            _host_ints("text2mel_generate_until", stop_pos, B, "stop position")
        order = np.argsort(np.where(sp < 0, np.iinfo(np.int32).max, sp), kind="stable")

        def decode(Ls):
            sps = self._i32(sp[order])
            Y = self._empty(B, self.hp.max_T, self.hp.n_mels)
            P = self._empty(B, self.hp.max_T, dtype=torch.int32)
            n = self._empty(B, dtype=torch.int32)
            self._check(self._lib.dctts_text2mel_generate_until(self._h, _ptr(Ls), B, int(steps), _ptr(sps), int(tail),
                                                                _ptr(Y), _ptr(P), _ptr(n), self._stream()),
                        "dctts_text2mel_generate_until")
            return Y, P, n
        return self._decode_in_order(L, order, decode)

    def text2mel_generate_path(self, L, path, lengths=None, steps=0):
        """The decode along a caller's attention windows (include/dctts.h: dctts_text2mel_generate_path): frame j of
        utterance b runs under the window path[b, j] instead of the previous frame's argmax.  `path`: (B, S) integers,
        S <= max_T; `lengths`: (B,) frames per utterance in [1, steps], default all `steps`; `steps` defaults to S.
        Returns (Y, prev_hist, argmax_hist) as CUDA tensors in the caller's order: prev_hist is the path, argmax_hist the
        model's own argmax of every frame; rows >= lengths[b] are 0 in Y and -1 in both histories.  The utterances are
        decoded in the order of their lengths, so that those sharing a decode cluster end at similar frames."""
        # Every host-side step comes before L is copied to the device: that copy waits for earlier work on the stream,
        # and host work after it would leave the GPU idle.
        B = len(L)
        ph = _host(path).astype(np.int64)
        if ph.ndim != 2 or ph.shape[0] != B:
            raise DcttsError("text2mel_generate_path: path must be (B, steps) for %d utterances, got %s" % (B, ph.shape))
        steps = int(steps) or ph.shape[1]
        if not 1 <= steps <= min(ph.shape[1], self.hp.max_T):
            raise DcttsError("text2mel_generate_path: steps %d outside [1, %d]" % (steps, min(ph.shape[1], self.hp.max_T)))
        # the library sees the utterances sorted: only here can a refusal name them in the caller's order
        n = np.full(B, steps, np.int64) if lengths is None else \
            _host_ints("text2mel_generate_path", lengths, B, "length", 1, steps)
        ph = ph[:, :steps]
        out = np.argwhere((np.arange(steps) < n[:, None]) & ((ph < 0) | (ph >= self.hp.max_N)))
        if out.size:
            b, j = out[0]
            raise DcttsError("text2mel_generate_path: utterance %d has window %d at frame %d outside [0, %d)"
                             % (b, ph[b, j], j, self.hp.max_N))
        order = np.argsort(n, kind="stable")
        ps = np.ascontiguousarray(ph[order], np.int32)
        ns = np.ascontiguousarray(n[order], np.int32)

        def decode(Ls):
            # host arrays: the entry point stages them itself, without waiting for earlier work on the stream
            Y = self._empty(B, self.hp.max_T, self.hp.n_mels)
            P = self._empty(B, self.hp.max_T, dtype=torch.int32)
            M = self._empty(B, self.hp.max_T, dtype=torch.int32)
            self._check(self._lib.dctts_text2mel_generate_path_host(self._h, _ptr(Ls), B, steps, C.c_void_p(ps.ctypes.data),
                                                                    C.c_void_p(ns.ctypes.data), _ptr(Y), _ptr(P), _ptr(M),
                                                                    self._stream()),
                        "dctts_text2mel_generate_path_host")
            return Y, P, M
        return self._decode_in_order(L, order, decode)

    def _decode_in_order(self, L, order, decode):
        """decode(Ls) on the texts L (B, max_N) taken in `order`, its (B, ...) CUDA outputs returned in the caller's order.
        decode_history reads the decode's own order from _decode_order."""
        L = self._i32(L)
        perm = None if np.array_equal(order, np.arange(len(order))) else torch.as_tensor(order, device=self.device)
        outs = decode(L if perm is None else L.index_select(0, perm).contiguous())
        self._decode_order = order
        if perm is None:
            return outs
        res = tuple(torch.empty_like(t) for t in outs)
        for r, t in zip(res, outs):
            r[perm] = t
        return res

    def _align_inputs(self, who, B, T, lengths, ends):
        """Host int32 lengths (default all T) and text ends (B,); the entry points check their ranges, naming the utterance."""
        n = np.full(B, T) if lengths is None else _host_ints(who, lengths, B, "length")
        return np.ascontiguousarray(n, np.int32), np.ascontiguousarray(_host_ints(who, ends, B, "text end"), np.int32)

    def _align_outputs(self, B, N, T):
        return (self._empty(B, T, dtype=torch.int32), self._empty(B, T, dtype=torch.int32),
                self._empty(B, N, dtype=torch.int32), self._empty(B, dtype=torch.float64))

    def align_search(self, alignments, lengths, ends):
        """The aligner's search alone (include/dctts.h: dctts_align_search) on alignments (B, N, T): for utterance b, the
        best monotonic path over lengths[b] frames ending at text position ends[b].  Returns CUDA tensors (path, chars,
        durations, score): path (B, T) the window of every frame as text2mel_generate_path takes it, chars (B, T) the
        character of every frame (both -1 past lengths[b]), durations (B, N) frames per text position, score (B,) float64
        the path's summed log-attention."""
        A = self._f32(alignments)
        if A.dim() != 3:
            raise DcttsError("align_search: alignments must be (B, N, T), got shape %s" % (tuple(A.shape),))
        B, N, T = A.shape
        n, e = self._align_inputs("align_search", B, T, lengths, ends)
        path, chars, dur, score = self._align_outputs(B, N, T)
        self._check(self._lib.dctts_align_search(self._h, _ptr(A), B, N, T, C.c_void_p(n.ctypes.data), C.c_void_p(e.ctypes.data),
                                                 _ptr(path), _ptr(chars), _ptr(dur), _ptr(score), self._stream()),
                    "dctts_align_search")
        return path, chars, dur, score

    def text2mel_align(self, L, mels, lengths=None, ends=None, want_alignments=False):
        """Align recorded speech to its text (include/dctts.h: dctts_text2mel_align): the teacher-forced Text2Mel front
        on L (B, max_N) and the recorded mels (B, T, n_mels), T <= max_T, then align_search on its dense attention.
        `lengths`: (B,) frames per recording, default all T; mels rows at and past them must be zeros, as
        load_spectrograms_batch writes them.  `ends`: (B,) text ends, default the EOS positions of L
        (data_load.eos_positions); an utterance without EOS is refused.  Returns CUDA tensors (path, chars, durations,
        score) as align_search does, and the alignments (B, max_N, T) when `want_alignments`."""
        from .data_load import eos_positions
        # Every host-side step comes before L is copied to the device (text2mel_generate_path explains why)
        Lh = _host(L)
        if Lh.ndim != 2 or Lh.shape[1] != self.hp.max_N:
            raise DcttsError("text2mel_align: L must be (B, max_N=%d), got shape %s" % (self.hp.max_N, Lh.shape))
        B, N = Lh.shape
        ms = tuple(mels.shape)
        if len(ms) != 3 or ms[0] != B or ms[2] != self.hp.n_mels or not 1 <= ms[1] <= self.hp.max_T:
            raise DcttsError("text2mel_align: mels must be (B=%d, T <= max_T=%d, n_mels=%d), got shape %s"
                             % (B, self.hp.max_T, self.hp.n_mels, ms))
        T = ms[1]
        n, e = self._align_inputs("text2mel_align", B, T, lengths, eos_positions(Lh) if ends is None else ends)
        L, mels = self._i32(Lh), self._f32(mels)
        path, chars, dur, score = self._align_outputs(B, N, T)
        A = self._empty(B, N, T) if want_alignments else None
        self._check(self._lib.dctts_text2mel_align(self._h, _ptr(L), _ptr(mels), B, T, C.c_void_p(n.ctypes.data),
                                                   C.c_void_p(e.ctypes.data), _ptr(path), _ptr(chars), _ptr(dur), _ptr(score),
                                                   _ptr(A), self._stream()), "dctts_text2mel_align")
        return (path, chars, dur, score, A) if want_alignments else (path, chars, dur, score)

    def mcd_dtw(self, X, nx, Y, ny, K=24, want_path=False):
        """Mel-cepstral distortion along a DTW alignment (include/dctts.h: dctts_mcd_dtw) between X[b, :nx[b]] and
        Y[b, :ny[b]], X (B, Tx, n_mels) and Y (B, Ty, n_mels) dB-normalised mels (Text2Mel's output, load_spectrograms's
        mels), using cepstral coefficients 1 .. K of an orthonormal DCT of the log mel amplitudes.  `nx`, `ny`: (B,)
        frames per sequence, read on the host.  Returns CUDA tensors (mcd (B,) float64, pairs (B,) int32: the cells on
        the path), and the path (B, Tx + Ty - 1, 2) int32 of (i, j) from (0, 0), -1 past pairs[b], when `want_path`.
        An MFCC-style distortion, not comparable to published (SPTK / WORLD) MCD figures."""
        X, Y = self._f32(X), self._f32(Y)
        M = self.hp.n_mels
        if X.dim() != 3 or X.shape[2] != M:
            raise DcttsError("mcd_dtw: X must be (B, Tx, n_mels=%d), got shape %s" % (M, tuple(X.shape)))
        B, Tx = X.shape[0], X.shape[1]
        if Y.dim() != 3 or Y.shape[0] != B or Y.shape[2] != M:
            raise DcttsError("mcd_dtw: Y must be (B=%d, Ty, n_mels=%d), got shape %s" % (B, M, tuple(Y.shape)))
        Ty = Y.shape[1]
        if B < 1 or Tx < 1 or Ty < 1:
            raise DcttsError("mcd_dtw: empty batch or sequences: X %s, Y %s" % (tuple(X.shape), tuple(Y.shape)))
        if not 1 <= int(K) <= M - 1:
            raise DcttsError("mcd_dtw: K must be in [1, n_mels - 1 = %d], got %d" % (M - 1, int(K)))
        nxh = np.ascontiguousarray(_host_ints("mcd_dtw", nx, B, "X length"), np.int32)
        nyh = np.ascontiguousarray(_host_ints("mcd_dtw", ny, B, "Y length"), np.int32)
        self._set_vocoder_params()
        mcd = self._empty(B, dtype=torch.float64)
        pairs = self._empty(B, dtype=torch.int32)
        path = self._empty(B, Tx + Ty - 1, 2, dtype=torch.int32) if want_path else None
        self._check(self._lib.dctts_mcd_dtw(self._h, _ptr(X), Tx, C.c_void_p(nxh.ctypes.data), _ptr(Y), Ty,
                                            C.c_void_p(nyh.ctypes.data), B, int(K), _ptr(mcd), _ptr(pairs), _ptr(path),
                                            self._stream()), "dctts_mcd_dtw")
        return (mcd, pairs, path) if want_path else (mcd, pairs)

    _HISTORY = {"audioenc": 0, "audiodec": 1, "R": 2, "KV": 3, "Y": 4, "windows": 5}

    def decode_history(self, what, layer=0):
        """Test aid (include/dctts.h: dctts_decode_history): the decode state of the last text2mel_generate(_until, _path) on
        this engine, in that call's order of the utterances.  what: "audioenc" / "audiodec" (block `layer`'s output rows
        (B, T, C), the last AudioDec block's are the logits), "R" (B, T, 2d), "KV" (B, N, 2d), "Y" (B, T, n_mels) or
        "windows" (B, T) int32.  Returns (tensor, joined): joined is True when the rows are hi + lo of the split-fp16 planes
        the decode kept instead of float32 rows.  Raises DcttsError when the engine's decode buffers were written by anything
        else since that call."""
        from .arch import audiodec_layers, audioenc_layers
        if what not in self._HISTORY:
            raise DcttsError("decode_history: `what` must be one of %s" % sorted(self._HISTORY))
        order = getattr(self, "_decode_order", None)
        if order is None:
            raise DcttsError("decode_history: no generation has run on this engine")
        h = self.hp
        B, T = len(order), h.max_T
        net = {"audioenc": audioenc_layers, "audiodec": audiodec_layers}.get(what)
        if net is not None and not 0 <= layer < len(net()):
            raise DcttsError("decode_history: %s has no block %d" % (what, layer))
        shape = {"audioenc": (B, T, h.d), "audiodec": (B, T, net()[layer].cout if net else 0), "R": (B, T, 2 * h.d),
                 "KV": (B, h.max_N, 2 * h.d), "Y": (B, T, h.n_mels), "windows": (B, T)}[what]
        out = self._empty(*shape, dtype=torch.int32 if what == "windows" else torch.float32)
        joined = C.c_int32(0)
        self._check(self._lib.dctts_decode_history(self._h, self._HISTORY[what], int(layer), _ptr(out), out.numel(),
                                                   C.byref(joined), self._stream()), "dctts_decode_history")
        res = torch.empty_like(out)
        res[torch.as_tensor(order, device=self.device)] = out
        return res, bool(joined.value)

    _CHAIN_NETS = {"textenc": 0, "audioenc": 1, "audiodec": 2, "ssrn": 3, "attention": 4}

    def chain_history(self, net, layer=0, what="output"):
        """Test aid (include/dctts.h: dctts_chain_history; needs set_option("chain_history", 1) before the call it reads):
        the rows the last call's full-sequence chain of `net` ("textenc", "audioenc", "audiodec", "ssrn", or "attention",
        whose output is R) left.  what: "output" (block `layer`'s) or "input" (the first block's, as its kernel read it).
        Returns (tensor (B, L, C) float32 in the caller's order, joined): joined is True when the rows are hi + lo of the
        split-fp16 planes the chain kept.  Raises DcttsError, naming the reason, when the last call did not keep them."""
        if net not in self._CHAIN_NETS or what not in ("output", "input"):
            raise DcttsError("chain_history: net must be one of %s and what 'output' or 'input'" % sorted(self._CHAIN_NETS))
        args = (self._h, self._CHAIN_NETS[net], int(layer), int(what == "input"))
        B, L, Cc = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._check(self._lib.dctts_chain_history_shape(*args, C.byref(B), C.byref(L), C.byref(Cc)), "dctts_chain_history")
        out = self._empty(B.value, L.value, Cc.value)
        joined = C.c_int32(0)
        self._check(self._lib.dctts_chain_history(*args, _ptr(out), out.numel(), C.byref(joined), self._stream()),
                    "dctts_chain_history")
        return out, bool(joined.value)

    def _set_vocoder_params(self, hop=None, win=None, power=None):
        """The hyperparameters' vocoder constants on the handle, with `hop`, `win` and `power` instead when given."""
        h = self.hp
        self._check(self._lib.dctts_set_vocoder_params(self._h, int(hop or h.hop_length), int(win or h.win_length),
                                                       float(h.power if power is None else power), float(h.max_db),
                                                       float(h.ref_db), float(h.preemphasis), int(h.n_iter)),
                    "dctts_set_vocoder_params")

    def spectrogram2wav(self, mag, n_iter=-1, lengths=None, momentum=0.0, convergence=False):
        """utils.py:67-94 for a batch: mag (B, T, F) in [0,1] -> (untrimmed wav (B, hop*(T-1)) CUDA tensor,
        trim (B, 2) int32 numpy [start, end) as librosa.effects.trim would keep).  Every call goes through
        dctts_spectrogram2wav_momentum (include/dctts.h), so its errors name that entry point.
        `lengths`: optional (B,) magnitude frames per utterance, 2 <= lengths[b] <= T: wav[b, :hop*(lengths[b]-1)] and
        trim[b] are what this call gives for mag[b:b+1, :lengths[b]] alone, bit for bit, the rest of wav[b] is 0, and mag
        rows past lengths[b] are never read.
        `momentum`: the fast Griffin-Lim update of librosa's griffinlim(momentum=...); 0 is the reference's plain update.
        Above 1 it warns, as librosa does; a negative one is refused.
        `convergence=True` also returns the spectral convergence ||S - |STFT(x_i)||| / ||S|| of every iteration i = 0 ..
        n_iter, (B, n_iter + 1) float64 CUDA tensor, as a third value."""
        mag = self._f32(mag)
        if mag.dim() == 2:
            mag = mag[None]
        B, T, F = mag.shape
        h = self.hp
        self._set_vocoder_params()
        wav = self._empty(B, h.hop_length * (T - 1))
        trim = np.zeros((B, 2), np.int32)
        n = None
        if lengths is not None:
            n = np.ascontiguousarray(_host_ints("spectrogram2wav", lengths, B, "length"), np.int32)
        momentum = float(momentum)
        if momentum > 1:
            warnings.warn("Griffin-Lim with momentum=%g > 1 can be unstable. Proceed with caution!" % momentum, stacklevel=2)
        iters = h.n_iter if n_iter < 0 else int(n_iter)
        conv = self._empty(B, iters + 1, dtype=torch.float64) if convergence else None
        self._check(self._lib.dctts_spectrogram2wav_momentum(
            self._h, _ptr(mag), B, T, None if n is None else n.ctypes.data_as(C.c_void_p), iters, momentum, _ptr(wav),
            trim.ctypes.data_as(C.c_void_p), _ptr(conv), self._stream()), "dctts_spectrogram2wav_momentum")
        return (wav, trim, conv) if convergence else (wav, trim)

    def vocoder_stream(self, B, T_cap=None, n_iter=-1, momentum=0.0):
        """Streaming Griffin-Lim (include/dctts.h: dctts_vocoder_stream_*) for B utterances of at most T_cap magnitude
        frames (default hp.r * hp.max_T), with spectrogram2wav's n_iter and momentum.  Returns a VocoderStream:
        push(mag, counts, final) appends counts[b] rows of mag (B, R, F) to utterance b and returns, per utterance, the
        float32 numpy samples that became final; close() returns the trims (B, 2) as spectrogram2wav reports them.  The
        samples of one utterance concatenate to spectrogram2wav's untrimmed waveform of its frames, bit for bit when
        a single push delivers them all."""
        T_cap = int(T_cap or self.hp.r * self.hp.max_T)
        momentum = float(momentum)
        if momentum > 1:
            warnings.warn("Griffin-Lim with momentum=%g > 1 can be unstable. Proceed with caution!" % momentum, stacklevel=2)
        self._set_vocoder_params()
        return VocoderStream(self, int(B), T_cap, int(n_iter), momentum)

    def synthesis_stream(self, L, stop_pos=None, tail=0, chunk=16, n_iter=-1, momentum=0.0):
        """Streaming synthesis from text (include/dctts.h: dctts_synth_stream_*): the until-EOS decode of the texts L
        (B, max_N) starts now, and poll() returns audio while it is still running.  stop_pos and tail are
        text2mel_generate_until's, n_iter and momentum spectrogram2wav's; each utterance's mel frames are turned into
        audio in chunks of `chunk` frames on a fixed grid, so the samples do not depend on when poll() runs.  Returns a
        SynthesisStream: poll(wait=True) gives B float32 numpy arrays of new samples (iterating yields them until every
        utterance is done), close() gives (lengths, trims) as text2mel_generate_until and spectrogram2wav report them.
        The utterances are decoded in the order of their stop positions, as text2mel_generate_until does; everything
        comes back in the caller's order."""
        from .data_load import eos_positions
        if tail < 0:
            raise DcttsError("synthesis_stream: tail must be >= 0")
        L = self._i32(L)
        B = L.shape[0]
        sp = eos_positions(L.cpu().numpy()) if stop_pos is None else _host_ints("synthesis_stream", stop_pos, B, "stop position")
        order = np.argsort(np.where(sp < 0, np.iinfo(np.int32).max, sp), kind="stable")
        momentum = float(momentum)
        if momentum > 1:
            warnings.warn("Griffin-Lim with momentum=%g > 1 can be unstable. Proceed with caution!" % momentum, stacklevel=2)
        self._set_vocoder_params()
        return SynthesisStream(self, L, order, sp, int(tail), int(chunk), int(n_iter), momentum)

    def ssrn_halo(self):
        """(left, right): the mel frames of context SSRN needs on each side of a run of frames (dctts_ssrn_halo)."""
        left, right = C.c_int32(), C.c_int32()
        self._check(self._lib.dctts_ssrn_halo(self._h, C.byref(left), C.byref(right)), "dctts_ssrn_halo")
        return left.value, right.value

    def ssrn_windows(self, Y, starts, counts, lengths):
        """Test aid (include/dctts.h: dctts_ssrn_windows): a synthesis stream's windowed SSRN on Y (B, T, n_mels).
        Utterance b commits mel rows [starts[b], starts[b] + counts[b]) at length lengths[b]; returns Z (B, 4 max(counts),
        F) with each utterance's 4 counts[b] sigmoid rows first and zeros after."""
        Y = self._f32(Y)
        B, T, _ = Y.shape
        st = np.ascontiguousarray(_host_ints("ssrn_windows", starts, B, "start"), np.int32)
        ct = np.ascontiguousarray(_host_ints("ssrn_windows", counts, B, "count", 1), np.int32)
        n = np.ascontiguousarray(_host_ints("ssrn_windows", lengths, B, "length", 1, T), np.int32)
        ld = int(ct.max())
        Z = torch.zeros(B, self.hp.r * ld, self.F, device=self.device)
        self._check(self._lib.dctts_ssrn_windows(self._h, _ptr(Y), B, T, st.ctypes.data_as(C.c_void_p),
                                                 ct.ctypes.data_as(C.c_void_p), n.ctypes.data_as(C.c_void_p), _ptr(Z), ld,
                                                 self._stream()), "dctts_ssrn_windows")
        return Z

    def vocoder_momentum_step(self, wav, S, E, X, momentum, partials=None, hop=None, win=None):
        """Test aid (include/dctts.h: dctts_vocoder_momentum_step): ONE fast Griffin-Lim phase step on caller CUDA tensors.
        wav (B, Ly) and S (B, T, F) float32 in; E (B, T, F) complex64 holds est_{i-1} on entry and est_i on return;
        X (B, T, F) complex64 out; partials: optional (B, T) float32 out, each frame's sum (S - |est_i|)^2."""
        hop = int(hop or self.hp.hop_length)
        self._set_vocoder_params(hop, win)
        B, T = S.shape[0], S.shape[1]
        want = [(wav, (B, hop * (T - 1)), torch.float32), (S, (B, T, self.F), torch.float32),
                (E, (B, T, self.F), torch.complex64), (X, (B, T, self.F), torch.complex64)]
        if partials is not None:
            want.append((partials, (B, T), torch.float32))
        _require_tensors("vocoder_momentum_step", want)
        self._check(self._lib.dctts_vocoder_momentum_step(self._h, B, T, _ptr(wav), _ptr(S), _ptr(E), _ptr(X), float(momentum),
                                                          _ptr(partials), self._stream()), "dctts_vocoder_momentum_step")
        return X

    def vocoder_stage(self, stage, x, out, S=None, hop=None, win=None, power=None):
        """Test aid (include/dctts.h: dctts_vocoder_stage): ONE stage of spectrogram2wav on caller CUDA tensors, with the
        hyperparameters' vocoder constants except `hop`, `win` and `power` when given.  Ly = hop (T - 1), F = 1 + n_fft/2:
          0 prepare     x = mag (B, T, F) float32                -> out = X (B, T, F) complex64
          1 istft       x = X (B, T, F) complex64                -> out = wav (B, Ly) float32
          2 stft_phase  x = wav (B, Ly), S = (B, T, F) float32   -> out = X (B, T, F) complex64
          3 deemph      x = out = wav (B, Ly), in place
          4 energies    x = wav (B, Ly)                          -> out = mse (B, 1 + Ly // 512) float32
        Tensors must be contiguous (they may be views into larger buffers).  Returns the trims (B, 2) int32 numpy for
        stage 4 (as spectrogram2wav reports them), else out."""
        hop = int(hop or self.hp.hop_length)
        self._set_vocoder_params(hop, win, power)
        f32, c64 = torch.float32, torch.complex64
        B = x.shape[0]
        if stage in (0, 1):
            T = x.shape[1]
        elif stage == 2:
            if S is None or S.dim() != 3:
                raise DcttsError("vocoder_stage: stage 2 (stft_phase) needs S (B, T, F)")
            T = S.shape[1]
        else:
            T = x.shape[1] // hop + 1
        Ly, F = hop * (T - 1), self.F
        want = {0: [(x, (B, T, F), f32), (out, (B, T, F), c64)],
                1: [(x, (B, T, F), c64), (out, (B, Ly), f32)],
                2: [(x, (B, Ly), f32), (S, (B, T, F), f32), (out, (B, T, F), c64)],
                3: [(x, (B, Ly), f32), (out, (B, Ly), f32)],
                4: [(x, (B, Ly), f32), (out, (B, 1 + Ly // 512), f32)]}.get(stage, [])
        _require_tensors("vocoder_stage %d" % stage, want)
        trim = np.zeros((B, 2), np.int32)
        self._check(self._lib.dctts_vocoder_stage(self._h, int(stage), B, T, _ptr(x), _ptr(S), _ptr(out),
                                                  trim.ctypes.data_as(C.POINTER(C.c_int32)), self._stream()),
                    "dctts_vocoder_stage")
        return trim if stage == 4 else out

    def feature_stage(self, stage, out, out2=None, wav=None, segments=None, r=None, sr=None):
        """Test aid (include/dctts.h: dctts_feature_stage): ONE stage of load_spectrograms_batch on caller CUDA tensors, with
        the hyperparameters' vocoder constants and the feature tables for `sr` (default hp.sr).  wav: packed 1-D float32 or
        int16 CUDA samples.  F = 1 + n_fft/2:
          0 energies  segments = (B + 1) sample offsets          -> out = mse, sum_b (1 + n_b // 512) float32
          1 spectra   segments = (B, 2) (first sample, length)   -> out = mag (B, r T_b, F), out2 = mel (B, T_b, n_mels)
          2 tables                                               -> out = mel weights (n_mels, F), out2 = window (win)
        Stage 1 writes only utterance b's rows t < 1 + length // hop of mag and t / r (t % r == 0) of mel.  Returns the
        trims (B, 2) int32 numpy for stage 0, the filter ranges (n_mels, 2) int32 numpy for stage 2, else out."""
        h = self.hp
        r = int(r or h.r)
        self._set_vocoder_params()
        f32 = torch.float32
        seg = None if segments is None else np.ascontiguousarray(np.asarray(segments).reshape(-1), dtype=np.int64)
        dtype, B, T_b = 0, 1, 0
        if stage in (0, 1):
            if wav is None or seg is None:
                raise DcttsError("feature_stage %d: needs wav and segments" % stage)
            dtype = 1 if wav.dtype == torch.int16 else 0
            _require_tensors("feature_stage %d" % stage, [(wav, (wav.numel(),), wav.dtype)])
            B = seg.size - 1 if stage == 0 else seg.size // 2
        if stage == 0:
            n = np.diff(seg)
            want = [(out, (int((1 + n // 512).sum()),), f32)]
        elif stage == 1:
            T_b = out2.shape[1]
            want = [(out, (B, r * T_b, self.F), f32), (out2, (B, T_b, h.n_mels), f32)]
        else:
            want = [(out, (h.n_mels, self.F), f32), (out2, (int(h.win_length),), f32)]
        _require_tensors("feature_stage %d" % stage, want)
        host = np.zeros((h.n_mels if stage == 2 else B, 2), np.int32)
        self._check(self._lib.dctts_feature_stage(
            self._h, int(stage), int(sr or h.sr), _ptr(wav), dtype,
            None if seg is None else seg.ctypes.data_as(C.POINTER(C.c_int64)), B, r, T_b, _ptr(out), _ptr(out2),
            host.ctypes.data_as(C.POINTER(C.c_int32)), self._stream()), "dctts_feature_stage")
        return out if stage == 1 else host

    def get_spectrograms(self, wav, sr=None):
        """utils.py:20-65 from a loaded waveform (1-D float32, hp.sr): -> (mel (T, n_mels), mag (T, F)) CUDA tensors and
        the [start, end) sample range librosa.effects.trim keeps."""
        h = self.hp
        wav = self._f32(wav).reshape(-1)
        n = wav.numel()
        self._set_vocoder_params()
        cap = 1 + n // h.hop_length
        mel = self._empty(cap, h.n_mels)
        mag = self._empty(cap, self.F)
        t = C.c_int32(0)
        trim = (C.c_int32 * 2)()
        self._check(self._lib.dctts_get_spectrograms(self._h, _ptr(wav), n, int(sr or h.sr), _ptr(mel), _ptr(mag), cap,
                                                     C.byref(t), trim, self._stream()), "dctts_get_spectrograms")
        return mel[:t.value], mag[:t.value], (int(trim[0]), int(trim[1]))

    def _pack(self, wavs, what):
        """1-D int16 / float32 waveforms -> (device tensor of them back to back, 1 if int16 else 0, int64 offsets (B+1)),
        through one pinned host buffer and one copy.  int16 stays int16 when every member is int16."""
        arrs = [np.asarray(w).reshape(-1) for w in wavs]
        if not arrs:
            raise DcttsError("%s: empty batch" % what)
        pcm = all(a.dtype == np.int16 for a in arrs)
        if not pcm:
            arrs = [a.astype(np.float32) / np.float32(32768.0) if a.dtype == np.int16 else np.asarray(a, np.float32) for a in arrs]
        offsets = np.zeros(len(arrs) + 1, np.int64)
        offsets[1:] = np.cumsum([a.size for a in arrs])
        host = torch.empty(int(offsets[-1]), dtype=torch.int16 if pcm else torch.float32, pin_memory=True)
        hv = host.numpy()
        for b, a in enumerate(arrs):
            hv[offsets[b]:offsets[b + 1]] = a
        return host.to(self.device, non_blocking=True), 1 if pcm else 0, offsets

    def _resample(self, wav, dtype, offsets, rates, sr_out, out=None):
        """dctts_resample_batch on packed device samples: -> (float32 outputs back to back, int64 offsets (B+1))."""
        B = len(offsets) - 1
        rates = np.ascontiguousarray(rates, np.int32)
        if rates.shape != (B,):
            raise DcttsError("resample: %d rates for %d utterances" % (rates.size, B))
        ratio = sr_out / np.maximum(rates, 1).astype(np.float64)
        cap = int(np.ceil(np.diff(offsets) * np.where(rates == sr_out, 1.0, ratio)).sum())
        if out is None or out.numel() < cap:
            out = self._empty(max(cap, 1))
        out_offsets = np.zeros(B + 1, np.int64)
        i64p = C.POINTER(C.c_int64)
        self._check(self._lib.dctts_resample_batch(
            self._h, _ptr(wav), dtype, offsets.ctypes.data_as(i64p), rates.ctypes.data_as(C.POINTER(C.c_int32)), B, int(sr_out),
            _ptr(out), out.numel(), out_offsets.ctypes.data_as(i64p), self._stream()), "dctts_resample_batch")
        return out, out_offsets

    def resample_batch(self, wavs, rates, sr_out=None):
        """What librosa.load(..., sr=sr_out) does after decoding (librosa 0.6 core.resample, res_type='kaiser_best',
        fix=True) for a list of 1-D int16 (PCM, value / 32768) or float32 waveforms at their native `rates`: one copy to
        the device, one kernel, no synchronisation.  Returns the float32 results as a list of CUDA tensors (views of one
        buffer); an utterance already at sr_out (default hp.sr) comes back unchanged, as float32."""
        wav, dtype, offsets = self._pack(wavs, "resample_batch")
        out, oo = self._resample(wav, dtype, offsets, rates, int(sr_out or self.hp.sr))
        return [out[oo[b]:oo[b + 1]] for b in range(len(oo) - 1)]

    def load_spectrograms_batch(self, wavs, sr=None, t_capacity=None, rates=None):
        """utils.py:147-162 for a list of 1-D int16 (PCM, value / 32768) or float32 waveforms, as ONE bucketed
        batch: the waveforms cross to the device in one copy from a pinned buffer (int16 stays int16 when every member
        is int16), two kernels compute all the features, and the call synchronises once.  `rates` gives each waveform's
        native sample rate (None: all at `sr`, default hp.sr); when some differ, one more kernel first resamples the
        batch to `sr` as librosa.load(..., sr=hp.sr) does (`resample_batch`) into a buffer the engine keeps, and the
        features read that.  Returns (mels (B, T_b, n_mels), mags (B, r T_b, F)) contiguous CUDA tensors zero-padded to
        the longest member, the reduced rows per utterance t (B,) int32 and the kept sample ranges trim (B, 2) int32
        (numpy; at `sr`).  `t_capacity` (reduced rows per utterance; default: enough for the untrimmed lengths) sizes
        the outputs."""
        h = self.hp
        sr = int(sr or h.sr)
        wav, dtype, offsets = self._pack(wavs, "load_spectrograms_batch")
        B = len(offsets) - 1
        if rates is not None and any(int(r) != sr for r in rates):
            self._rs_out, offsets = self._resample(wav, dtype, offsets, rates, sr, getattr(self, "_rs_out", None))
            wav, dtype = self._rs_out, 0
        if t_capacity is None:
            t_capacity = max(-(-(1 + int(n) // h.hop_length) // h.r) for n in np.diff(offsets))
        self._set_vocoder_params()
        mel = self._empty(B * t_capacity * h.n_mels)
        mag = self._empty(B * t_capacity * h.r * self.F)
        t = np.zeros(B, np.int32)
        trim = np.zeros((B, 2), np.int32)
        T_b = C.c_int32(0)
        i32p = C.POINTER(C.c_int32)
        self._check(self._lib.dctts_load_spectrograms_batch(
            self._h, _ptr(wav), dtype, offsets.ctypes.data_as(C.POINTER(C.c_int64)), B, sr, _ptr(mel),
            _ptr(mag), int(t_capacity), t.ctypes.data_as(i32p), trim.ctypes.data_as(i32p), C.byref(T_b), self._stream()),
            "dctts_load_spectrograms_batch")
        T_b = T_b.value
        mel = mel[:B * T_b * h.n_mels].view(B, T_b, h.n_mels)
        mag = mag[:B * h.r * T_b * self.F].view(B, h.r * T_b, self.F)
        return mel, mag, t, trim

    # ------------------------------------------------------------------ training step (BASELINE config 5)
    def train_init(self, B, dropout_rate=None):
        """Allocates the training workspace for batches of B utterances (train.py mode "train", num=1)."""
        rate = self.hp.dropout_rate if dropout_rate is None else dropout_rate
        self._check(self._lib.dctts_train_init(self._h, int(B), float(rate)), "dctts_train_init")

    def _text_mels(self, who, L, mels):
        L = self._i32(L); mels = self._f32(mels)
        if L.dim() != 2:
            raise DcttsError("%s: L must be (B, N), got shape %s" % (who, tuple(L.shape)))
        B = L.shape[0]
        if mels.dim() != 3 or mels.shape[0] != B or mels.shape[2] != self.hp.n_mels:
            raise DcttsError("%s: mels must be (B=%d, T, n_mels=%d), got shape %s" % (who, B, self.hp.n_mels, tuple(mels.shape)))
        return L, mels

    def _mels_mags(self, who, mels, mags):
        mels = self._f32(mels); mags = self._f32(mags)
        if mels.dim() != 3 or mels.shape[2] != self.hp.n_mels:
            raise DcttsError("%s: mels must be (B, T, n_mels=%d), got shape %s" % (who, self.hp.n_mels, tuple(mels.shape)))
        B, T = mels.shape[0], mels.shape[1]
        if tuple(mags.shape) != (B, self.hp.r * T, self.F):
            raise DcttsError("%s: mags must be (B, %d T, F) = %s for mels %s, got %s"
                             % (who, self.hp.r, (B, self.hp.r * T, self.F), tuple(mels.shape), tuple(mags.shape)))
        return mels, mags

    def train_step(self, L, mels, global_step=0, seed=0, lr=None, apply=True):
        """One Text2Mel optimiser step on L (B, N) int32 / mels (B, T, n_mels) at the batch's own shape -- a bucket padded
        to its longest member (trainer.bucketed_batches) or the fixed (max_N, max_T) -- up to N = hp.max_N, T = hp.max_T,
        or the capacity given to train_reserve:
        forward with dropout, losses (train.py:83-99), backward, clip, Adam (train.py:122-132).
        Returns {loss, loss_mels, loss_bd1, loss_att}."""
        L, mels = self._text_mels("train_step", L, mels)
        B, N = L.shape
        out = (C.c_float * 4)()
        self._check(self._lib.dctts_train_step_shaped(self._h, _ptr(L), N, _ptr(mels), mels.shape[1], B, int(global_step),
                                                      int(seed) & 0xffffffff, float(self.hp.lr if lr is None else lr),
                                                      1 if apply else 0, out, self._stream()), "dctts_train_step")
        return {"loss": out[0], "loss_mels": out[1], "loss_bd1": out[2], "loss_att": out[3]}

    def train_init_ssrn(self, B, T=None, dropout_rate=None):
        """Training workspace for the SSRN trainer (train.py num=2): mels (B, T, n_mels) -> mags (B, 4T, F) for any T up
        to the capacity `T` (default hp.max_T).
        Measured parity: all 80 gradient tensors within 6e-6 of the autograd checker's (DESIGN.md 8e)."""
        rate = self.hp.dropout_rate if dropout_rate is None else dropout_rate
        self._check(self._lib.dctts_train_init_ssrn(self._h, int(B), int(self.hp.max_T if T is None else T), float(rate)),
                    "dctts_train_init_ssrn")

    def train_step_ssrn(self, mels, mags, global_step=0, seed=0, lr=None, apply=True):
        """One SSRN optimiser step on ground-truth mels (B, T, n_mels) / mags (B, 4T, F) at the batch's own T, up to the
        capacity of train_init_ssrn (train.py:69-72,100-108,122-132)."""
        mels, mags = self._mels_mags("train_step_ssrn", mels, mags)
        B, T = mels.shape[0], mels.shape[1]
        out = (C.c_float * 4)()
        self._check(self._lib.dctts_train_step_ssrn_shaped(self._h, _ptr(mels), _ptr(mags), B, T, int(global_step),
                                                           int(seed) & 0xffffffff, float(self.hp.lr if lr is None else lr),
                                                           1 if apply else 0, out, self._stream()), "dctts_train_step_ssrn")
        return {"loss": out[0], "loss_mags": out[1], "loss_bd2": out[2]}

    def train_eval(self, L, mels, seed=0, want=("Y", "alignments")):
        """The Text2Mel training graph evaluated on one batch without an update -- the reference's sess.run(g.alignments)
        or sess.run(g.merged) (train.py:100-104,156): the step's forward with its dropout mask at `seed`, and its losses at
        the batch's shape.  Same shapes as train_step.  The variables, Adam moments and the gradient arena are untouched.
        Returns ({loss, loss_mels, loss_bd1, loss_att}, {name: CUDA tensor}) for the names in `want`: "Y" (B, T, n_mels)
        and "alignments" (B, N, T)."""
        L, mels = self._text_mels("train_eval", L, mels)
        B, N = L.shape
        unknown = set(want) - {"Y", "alignments"}
        if unknown:
            raise DcttsError("train_eval: can return Y and alignments, not %s" % sorted(unknown))
        T = mels.shape[1]
        tensors = {}
        if "Y" in want:
            tensors["Y"] = self._empty(B, T, self.hp.n_mels)
        if "alignments" in want:
            tensors["alignments"] = self._empty(B, N, T)
        out = (C.c_float * 4)()
        self._check(self._lib.dctts_train_eval(self._h, _ptr(L), N, _ptr(mels), T, B, int(seed) & 0xffffffff, _ptr(tensors.get("Y")),
                                               _ptr(tensors.get("alignments")), out, self._stream()), "dctts_train_eval")
        return {"loss": out[0], "loss_mels": out[1], "loss_bd1": out[2], "loss_att": out[3]}, tensors

    def train_eval_ssrn(self, mels, mags, seed=0, want=("Z",)):
        """The SSRN counterpart of train_eval (train.py:115-118): returns ({loss, loss_mags, loss_bd2}, {"Z": (B, 4T, F)})."""
        mels, mags = self._mels_mags("train_eval_ssrn", mels, mags)
        B, T = mels.shape[0], mels.shape[1]
        unknown = set(want) - {"Z"}
        if unknown:
            raise DcttsError("train_eval_ssrn: can return Z, not %s" % sorted(unknown))
        tensors = {"Z": self._empty(B, self.hp.r * T, self.F)} if "Z" in want else {}
        out = (C.c_float * 4)()
        self._check(self._lib.dctts_train_eval_ssrn(self._h, _ptr(mels), _ptr(mags), B, T, int(seed) & 0xffffffff,
                                                    _ptr(tensors.get("Z")), out, self._stream()), "dctts_train_eval_ssrn")
        return {"loss": out[0], "loss_mags": out[1], "loss_bd2": out[2]}, tensors

    def train_reserve(self, N, T):
        """Grow the training workspace of the network being trained to at least N text positions (Text2Mel; ignored for
        SSRN) and T mel frames, so that train_step / train_step_ssrn accept batches up to that shape.  The variables, Adam
        moments and the gradient arena (train_grads' address) are kept.  Never shrinks; synchronises the device when it
        grows.  Past (max_N, max_T) the guided-attention loss covers the table's corner only (train.py:91-95)."""
        self._check(self._lib.dctts_train_reserve(self._h, int(N), int(T)), "dctts_train_reserve")

    def train_capacity(self):
        """(N_cap, T_cap) of the training workspace: (max_N, max_T) after train_init, (0, T) after train_init_ssrn, or what
        train_reserve grew it to."""
        n, t = C.c_int32(0), C.c_int32(0)
        self._check(self._lib.dctts_train_capacity(self._h, C.byref(n), C.byref(t)), "dctts_train_capacity")
        return n.value, t.value

    def train_apply(self, global_step, lr=None):
        self._check(self._lib.dctts_train_apply(self._h, int(global_step), float(self.hp.lr if lr is None else lr), self._stream()),
                    "dctts_train_apply")

    def train_grads(self):
        """The flat float32 gradient arena as a CUDA tensor sharing the library's memory (all-reduce it in a
        data-parallel job between train_step(apply=False) and train_apply)."""
        ptr, n = C.c_void_p(), C.c_int64(0)
        self._check(self._lib.dctts_train_grads(self._h, C.byref(ptr), C.byref(n)), "dctts_train_grads")

        class _View:
            __cuda_array_interface__ = {"shape": (n.value,), "typestr": "<f4", "data": (ptr.value, False), "version": 2}
        return torch.as_tensor(_View(), device=self.device)

    def train_tensor(self, name, what="param"):
        """Copy of a Text2Mel variable / its gradient / Adam m / v, in the TF variable's shape."""
        from .arch import param_shapes
        shape = param_shapes()[name]
        out = np.empty(shape, np.float32)
        self._check(self._lib.dctts_train_tensor(self._h, name.encode(), {"param": 0, "grad": 1, "m": 2, "v": 3}[what],
                                                 out.ctypes.data_as(C.c_void_p), out.size), "dctts_train_tensor(%s)" % name)
        return out

    def train_set_tensor(self, name, array, what="param"):
        """Upload a variable / Adam m / Adam v of the network being trained from the TF layout (resume)."""
        from .arch import param_shapes
        a = np.ascontiguousarray(array, dtype=np.float32)
        if tuple(a.shape) != tuple(param_shapes()[name]):
            raise DcttsError("train_set_tensor(%s): shape %s, expected %s" % (name, a.shape, param_shapes()[name]))
        self._check(self._lib.dctts_train_set_tensor(self._h, name.encode(), {"param": 0, "m": 2, "v": 3}[what],
                                                     a.ctypes.data_as(C.c_void_p), a.size), "dctts_train_set_tensor(%s)" % name)

    def refresh_synthesis(self):
        """Synthesise from the variables being trained (include/dctts.h: dctts_refresh_synthesis): packs the wgmma weight
        planes and the persistent decode's weight stream again on the device, so that this handle computes what a fresh
        handle loaded with the same variables computes, on the same kernels.  Training state is untouched; the next update
        (train_step with apply, train_apply, train_set_tensor of a variable, restore_training) makes the packing stale
        again.  A no-op when nothing changed since the last packing."""
        self._check(self._lib.dctts_refresh_synthesis(self._h, self._stream()), "dctts_refresh_synthesis")

    def restore_training(self, logdir, scope="Text2Mel"):
        """What tf.train.Supervisor does when `logdir` already holds a checkpoint (train.py:144): every variable of the
        network being trained, its Adam slots (`<name>/Adam`, `<name>/Adam_1`) and `gs/global_step` come back from the
        latest bundle, so a restarted run continues the Noam schedule and the Adam state instead of overwriting
        model_gs_001k from scratch.  Call after train_init / train_init_ssrn.  Returns the restored global step, or None
        when the directory holds no checkpoint."""
        from .arch import param_shapes
        from .checkpoint import latest_checkpoint, list_variables, load_checkpoint
        path = latest_checkpoint(logdir)
        if path is None:
            return None
        avail = {n for n, _, _ in list_variables(path)}
        names = [n for n in param_shapes() if n.startswith(scope + "/")]
        missing = [n for n in names if n not in avail]
        if missing:
            raise DcttsError("restore_training: %s lacks %s" % (path, ", ".join(missing[:3])))
        for n in names:
            want = [n] + [n + sfx for sfx in ("/Adam", "/Adam_1") if n + sfx in avail]
            t = load_checkpoint(path, want)
            self.train_set_tensor(n, t[n], "param")
            if n + "/Adam" in t:
                self.train_set_tensor(n, t[n + "/Adam"], "m")
            if n + "/Adam_1" in t:
                self.train_set_tensor(n, t[n + "/Adam_1"], "v")
        gs = 0
        if "gs/global_step" in avail:
            gs = int(load_checkpoint(path, ["gs/global_step"])["gs/global_step"])
        return gs

    def save_checkpoint(self, prefix, global_step, scope="Text2Mel"):
        """What `sv.saver.save(sess, logdir + '/model_gs_...')` writes at train.py:152 for the network being trained
        (`scope` "Text2Mel" or "SSRN"): every variable of the scope, its Adam slots (`<name>/Adam`, `<name>/Adam_1`),
        the optimiser's `beta1_power` / `beta2_power` (TF's Adam keeps beta^t as variables; a TF train-graph
        Saver.restore expects them) and `gs/global_step`, as a TF tensor bundle."""
        from .arch import param_shapes
        from .checkpoint import save_checkpoint
        out = {"gs/global_step": np.array(global_step, np.int32),
               "beta1_power": np.array(0.9 ** (global_step + 1), np.float32),      # after t applies TF holds beta^(t+1)
               "beta2_power": np.array(0.999 ** (global_step + 1), np.float32)}
        for name in param_shapes():
            if name.startswith(scope + "/"):
                out[name] = self.train_tensor(name, "param")
                out[name + "/Adam"] = self.train_tensor(name, "m")
                out[name + "/Adam_1"] = self.train_tensor(name, "v")
        return save_checkpoint(prefix, out)

    def save_text2mel_checkpoint(self, prefix, global_step):
        return self.save_checkpoint(prefix, global_step, "Text2Mel")

    def synthesize_host(self, L_host, Y_host=None, Z_host=None):
        """synthesize.py:45-57 with host (ideally pinned) tensors in and out."""
        L_host = torch.as_tensor(L_host, dtype=torch.int32).contiguous()
        B = L_host.shape[0]
        if Z_host is None:
            Z_host = torch.empty((B, self.hp.max_T * self.hp.r, self.F), dtype=torch.float32).pin_memory()
        if Y_host is None:
            Y_host = torch.empty((B, self.hp.max_T, self.hp.n_mels), dtype=torch.float32).pin_memory()
        self._check(self._lib.dctts_synthesize_host(self._h, _ptr(L_host), B, _ptr(Y_host), _ptr(Z_host)),
                    "dctts_synthesize_host")
        self._decode_order = np.arange(B)
        return Y_host, Z_host


_default = None


class VocoderStream:
    """One dctts_vocoder_stream on an engine (Engine.vocoder_stream).  Its output buffer is allocated at open and every
    call runs on the stream that was current then."""

    def __init__(self, eng, B, T_cap, n_iter, momentum):
        self._eng, self.B, self.T_cap = eng, B, T_cap
        self.ld = eng.hp.hop_length * (T_cap - 1)           # the most samples one push can commit for an utterance
        self._wav = eng._empty(B, self.ld)
        self._tstream = torch.cuda.current_stream(eng.device)
        self._stream = C.c_void_p(self._tstream.cuda_stream)
        vs = C.c_void_p()
        self._vs = None
        eng._check(eng._lib.dctts_vocoder_stream_open(eng._h, B, T_cap, n_iter, momentum, self._stream, C.byref(vs)),
                   "dctts_vocoder_stream_open")
        self._vs = vs
        eng._streams.add(self)

    def push(self, mag, counts, final=False):
        """mag (B, R, F) magnitudes (CUDA tensor or array), counts (B) rows of it per utterance, final: one flag or (B)
        flags -> B float32 numpy arrays of newly committed samples."""
        eng, B = self._eng, self.B
        if self._vs is None:
            raise DcttsError("dctts_vocoder_stream_push: the stream is closed")
        mag = eng._f32(mag)
        if mag.dim() != 3 or mag.shape[0] != B or mag.shape[2] != eng.F:
            raise DcttsError("dctts_vocoder_stream_push: expected mag (%d, R, %d), got %s" % (B, eng.F, tuple(mag.shape)))
        rows = np.ascontiguousarray(_host_ints("dctts_vocoder_stream_push", counts, B, "row count"), np.int32)
        fin = np.ascontiguousarray(np.broadcast_to(np.asarray(final, bool), (B,)), np.int32)
        n = np.zeros(B, np.int32)
        eng._check(eng._lib.dctts_vocoder_stream_push(
            self._vs, _ptr(mag), mag.shape[1], rows.ctypes.data_as(C.c_void_p), fin.ctypes.data_as(C.c_void_p),
            _ptr(self._wav), self.ld, n.ctypes.data_as(C.c_void_p)), "dctts_vocoder_stream_push")
        with torch.cuda.stream(self._tstream):
            host = self._wav[:, :int(n.max(initial=0))].cpu().numpy()
        return [host[b, :n[b]].copy() for b in range(B)]

    def close(self):
        """Frees the stream and returns the trims (B, 2) int32; DcttsError (the stream is freed all the same) when an
        utterance has not had its final push."""
        if self._vs is None:
            return None
        trim = np.zeros((self.B, 2), np.int32)
        vs, self._vs = self._vs, None
        self._eng._streams.discard(self)
        rc = self._eng._lib.dctts_vocoder_stream_close(vs, trim.ctypes.data_as(C.c_void_p))
        self._eng._check(rc, "dctts_vocoder_stream_close")
        return trim

    def _free(self):
        """Frees the stream without trims (Engine.close and garbage collection); its engine's handle is still open."""
        if getattr(self, "_vs", None) is not None:
            vs, self._vs = self._vs, None
            self._eng._streams.discard(self)
            self._eng._lib.dctts_vocoder_stream_close(vs, None)

    def __del__(self):
        self._free()


class SynthesisStream:
    """One dctts_synth_stream on an engine (Engine.synthesis_stream).  The decode runs on the stream that was current at
    open; the SSRN windows and the vocoder run on the library's own side stream."""

    def __init__(self, eng, L, order, stop_pos, tail, chunk, n_iter, momentum):
        self._eng, self.B = eng, L.shape[0]
        self._order = np.asarray(order)
        perm = torch.as_tensor(self._order, device=eng.device)
        self._L = L.index_select(0, perm).contiguous()          # kept alive while the decode reads it
        sps = np.ascontiguousarray(stop_pos[self._order], np.int32)
        self.ld = eng.hp.hop_length * (eng.hp.r * eng.hp.max_T - 1)
        self._wav = np.zeros((self.B, self.ld), np.float32)
        self.done = np.zeros(self.B, bool)
        self.frames = np.zeros(self.B, np.int32)             # decode frames published for each utterance at the last poll
        self.first_frames = None
        ss = C.c_void_p()
        self._ss = None
        eng._check(eng._lib.dctts_synth_stream_open(eng._h, _ptr(self._L), self.B, sps.ctypes.data_as(C.c_void_p), tail, chunk,
                                                    n_iter, momentum, eng._stream(), C.byref(ss)), "dctts_synth_stream_open")
        self._ss = ss
        eng._streams.add(self)

    def poll(self, wait=True):
        """B float32 numpy arrays (caller's order) of the samples committed since the last poll; with `wait`, blocks until
        there is something to return or every utterance is done."""
        if self._ss is None:
            raise DcttsError("dctts_synth_stream_poll: the stream is closed")
        B = self.B
        n, d, f = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B, np.int32)
        self._eng._check(self._eng._lib.dctts_synth_stream_poll(self._ss, int(bool(wait)), self._wav.ctypes.data_as(C.c_void_p),
                                                                self.ld, n.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p),
                                                                f.ctypes.data_as(C.c_void_p)),
                         "dctts_synth_stream_poll")
        out = [None] * B
        for i, b in enumerate(self._order):
            out[b] = self._wav[i, :n[i]].copy()
            self.done[b] = bool(d[i])
            self.frames[b] = f[i]
        return out

    def __iter__(self):
        while not self.done.all():
            yield self.poll()

    def close(self, outputs=False):
        """Waits for the decode, runs what is left and frees the stream.  Returns (lengths, trims) in the caller's order,
        as text2mel_generate_until and spectrogram2wav report them; with outputs=True also Y (B, max_T, n_mels) and Z
        (B, 4 max_T, F), CUDA tensors with rows past each length 0.  Sets first_frames: the decode frames published when
        each utterance's first chunk was pushed."""
        if self._ss is None:
            return None
        eng, B, h = self._eng, self.B, self._eng.hp
        n, trim, ff = np.zeros(B, np.int32), np.zeros((B, 2), np.int32), np.zeros(B, np.int32)
        Y = eng._empty(B, h.max_T, h.n_mels) if outputs else None
        Z = eng._empty(B, h.r * h.max_T, eng.F) if outputs else None
        ss, self._ss = self._ss, None
        eng._streams.discard(self)
        rc = eng._lib.dctts_synth_stream_close(ss, n.ctypes.data_as(C.c_void_p), trim.ctypes.data_as(C.c_void_p), _ptr(Y), _ptr(Z),
                                               ff.ctypes.data_as(C.c_void_p))
        eng._check(rc, "dctts_synth_stream_close")
        inv = np.empty(B, np.int64)
        inv[self._order] = np.arange(B)
        self.first_frames = ff[inv]
        res = (n[inv], trim[inv])
        if outputs:
            perm = torch.as_tensor(inv, device=eng.device)
            res += (Y.index_select(0, perm), Z.index_select(0, perm))
        return res

    def _free(self):
        """Frees the stream without outputs (Engine.close and garbage collection); its engine's handle is still open."""
        if getattr(self, "_ss", None) is not None:
            ss, self._ss = self._ss, None
            self._eng._streams.discard(self)
            self._eng._lib.dctts_synth_stream_close(ss, None, None, None, None, None)

    def __del__(self):
        self._free()


def get_engine():
    """The process-wide default engine (used by modules.py / networks.py wrappers)."""
    global _default
    if _default is None:
        import os
        _default = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    return _default


def set_engine(e):
    global _default
    _default = e
    return e
