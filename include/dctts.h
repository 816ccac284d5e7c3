/*
 * dctts.h -- C-ABI of the H100-native DC-TTS synthesis path (libdctts_b200.so).
 *
 * The reference (Kyubyong/dc_tts) has no FFI layer: its operator API is the set of
 * Python signatures in modules.py / networks.py and the Graph attributes fetched by
 * synthesize.py.  Each entry point below states the reference interface it replaces
 * (file:line under /root/reference).  INTEGRATION.md shows the ctypes binding.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *   - every tensor is float32, channels-last (B, time, C), dense unless an explicit
 *     leading dimension is passed; ids are int32, argmax outputs int64 (tf.argmax);
 *   - `x`/`out` pointers are DEVICE pointers on the handle's device, except in the
 *     `*_host` entry points, which take HOST pointers and do the copies themselves;
 *   - the caller owns all tensors; the handle owns weights, workspace and CUDA graphs;
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream);
 *   - every function returns 0 on success, non-zero on failure, never throws, and
 *     never falls back to a CPU implementation; dctts_last_error() describes the
 *     most recent failure on that handle (or the global one for create failures);
 *   - a handle is bound to one device and is not thread-safe.
 */
#ifndef DCTTS_H_
#define DCTTS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dctts_handle_s* dctts_handle;

/* Model hyper-parameters the kernels specialise on: reference hyperparams.py:19,27-32,38-40,14. */
typedef struct dctts_hparams {
    int32_t vocab_size;          /* len(hp.vocab) = 32 */
    int32_t e;                   /* hp.e = 128  */
    int32_t d;                   /* hp.d = 256  */
    int32_t c;                   /* hp.c = 512  */
    int32_t n_mels;              /* hp.n_mels = 80 */
    int32_t n_fft;               /* hp.n_fft = 2048 -> F = 1 + n_fft/2; the STFT kernels exist for 1024, 2048, 4096 */
    int32_t max_N;               /* hp.max_N = 180 */
    int32_t max_T;               /* hp.max_T = 210 */
    int32_t attention_win_size;  /* hp.attention_win_size = 3 */
    int32_t r;                   /* hp.r = 4 (SSRN upsampling = two stride-2 deconvs) */
} dctts_hparams;

/* ---- lifetime ------------------------------------------------------------------ */
/* Replaces Graph(mode="synthesize") construction + tf.Session() (train.py:22-80, synthesize.py:26-28). */
int dctts_create(const dctts_hparams* hp, int device, dctts_handle* out);
int dctts_destroy(dctts_handle h);
const char* dctts_last_error(dctts_handle h);      /* h may be NULL: last create() error */
const char* dctts_version(void);

/* ---- parameters ---------------------------------------------------------------- */
/* Replaces Saver.restore into TF variables (synthesize.py:31-41).  `tf_name` is the TF
 * variable name (SURVEY.md App. C), `data` a HOST float32 array of `shape[0..rank)`.
 * dctts_commit_params() packs the staged variables into the kernels' layouts and
 * uploads them; it fails if any variable of the path is missing or mis-shaped. */
int dctts_set_param(dctts_handle h, const char* tf_name, const float* data,
                    const int64_t* shape, int32_t rank);
int dctts_commit_params(dctts_handle h);
int64_t dctts_num_params(dctts_handle h);           /* committed scalar count, -1 on error */

/* ---- building blocks (reference modules.py) ------------------------------------ */
/* `scope` is the full variable scope, e.g. "Text2Mel/AudioEnc/HC_4". */

/* embed (modules.py:13-42): ids (B,N) int32 -> out (B,N,e); row 0 of the table reads as zeros. */
int dctts_embed(dctts_handle h, const char* scope, const int32_t* ids, int32_t B, int32_t N,
                float* out, void* stream);
/* normalize (modules.py:45-64): LN over the last axis with `scope`/{gamma,beta}, eps 1e-12. */
int dctts_normalize(dctts_handle h, const char* scope, const float* x, int64_t rows, int32_t C,
                    float* out, void* stream);
/* conv1d (modules.py:91-141, training=False): conv(k, rate, SAME|CAUSAL) + bias -> LN -> act.
 * k, Cin, Cout come from the committed kernel; act: 0 none, 1 relu.  x (B,L,Cin) -> out (B,L,Cout). */
int dctts_conv1d(dctts_handle h, const char* scope, const float* x, int32_t B, int32_t L,
                 int32_t rate, int32_t causal, int32_t act, float* out, void* stream);
/* hc (modules.py:143-197): conv to 2C -> split -> LN(H1),LN(H2) -> sigmoid(H1) -> H1*H2+(1-H1)*x. */
int dctts_hc(dctts_handle h, const char* scope, const float* x, int32_t B, int32_t L,
             int32_t rate, int32_t causal, float* out, void* stream);
/* conv1d_transpose (modules.py:199-247): stride-2, k=3, 'same' -> LN.  x (B,L,C) -> out (B,2L,C). */
int dctts_conv1d_transpose(dctts_handle h, const char* scope, const float* x, int32_t B, int32_t L,
                           float* out, void* stream);

/* ---- networks (reference networks.py) ------------------------------------------ */
/* TextEnc (networks.py:14-71): L (B,N) int32 -> K,V (B,N,d) each. */
int dctts_textenc(dctts_handle h, const int32_t* L, int32_t B, float* K, float* V, void* stream);
/* AudioEnc (networks.py:73-124): S (B,T,n_mels) -> Q (B,T,d). */
int dctts_audioenc(dctts_handle h, const float* S, int32_t B, int32_t T, float* Q, void* stream);
/* Attention (networks.py:126-155): Q (B,T,d), K,V (B,N,d) -> R (B,T,2d), alignments (B,N,T),
 * max_attentions (B,T) int64.  prev_max_attentions (B) int32 selects the monotonic window
 * [p, p+win) when `monotonic` != 0 (ignored otherwise, may be NULL).  alignments and
 * max_attentions may be NULL. */
int dctts_attention(dctts_handle h, const float* Q, const float* K, const float* V,
                    int32_t B, int32_t T, int32_t N, int32_t monotonic,
                    const int32_t* prev_max_attentions,
                    float* R, float* alignments, int64_t* max_attentions, void* stream);
/* AudioDec (networks.py:157-212): R (B,T,2d) -> Y_logits, Y (B,T,n_mels). Y_logits may be NULL. */
int dctts_audiodec(dctts_handle h, const float* R, int32_t B, int32_t T,
                   float* Y_logits, float* Y, void* stream);
/* SSRN (networks.py:214-292): Y (B,T,n_mels) -> Z_logits, Z (B,4T,F). Z_logits may be NULL. */
int dctts_ssrn(dctts_handle h, const float* Y, int32_t B, int32_t T,
               float* Z_logits, float* Z, void* stream);
/* dctts_ssrn and dctts_ssrn_ragged take any T, also above max_T (long-form synthesis): the buffers the SSRN chain runs in
 * grow in place to B x T mel frames (dctts_reserve_frames), and a T <= max_T call computes and launches what it did
 * before any growth. */
/* SSRN with a length per utterance.  lengths: (B) int32 DEVICE mel frames, 1 <= lengths[b] <= T (as
 * dctts_text2mel_generate_until writes them).  For each b, Z[b, :4 lengths[b]] and Z_logits[b, :4 lengths[b]] are
 * dctts_ssrn of Y[b:b+1, :lengths[b]] alone on the same kernel set, bit for bit; their rows past that are 0 (Z too).
 * Rows >= lengths[b] of Y are never read.  On the wgmma path (dctts_set_tensor_path 1) it is one launch per block over
 * the batch and no host sync; a length outside the range is clamped to [0, T] and no row outside the utterance's
 * [0, T) / [0, 4T) is touched.  On the fp32 path the lengths are copied to the host (a sync), a length outside the range
 * fails the call, and the chain runs once per utterance: that path's GEMM schedule depends on a launch's row count. */
int dctts_ssrn_ragged(dctts_handle h, const float* Y, int32_t B, int32_t T, const int32_t* lengths,
                      float* Z_logits, float* Z, void* stream);

/* ---- graph-level (reference train.py Graph, synthesize.py loop) ------------------ */
/* One sess.run of the synthesize graph (train.py:48-68 fetched at synthesize.py:48-52):
 * L (B,max_N), mels (B,max_T,n_mels), prev_max_attentions (B) ->
 * Y (B,max_T,n_mels), max_attentions (B,max_T) int64, alignments (B,max_N,max_T).
 * alignments may be NULL.  All rows are recomputed, as the reference does. */
int dctts_text2mel_forward(dctts_handle h, const int32_t* L, const float* mels,
                           const int32_t* prev_max_attentions, int32_t B,
                           float* Y, int64_t* max_attentions, float* alignments, void* stream);
/* The whole autoregressive loop of synthesize.py:45-54 on the device: TextEnc once, then
 * `steps` (<= max_T; 0 means max_T) incremental steps replayed from a CUDA graph, each
 * reproducing exactly what the reference's full-graph pass yields for row j (including
 * the re-application of step j's attention window to the 85-row AudioDec history).
 * Outputs: Y (B,max_T,n_mels); optional prev_hist (B,max_T) int32 = the
 * prev_max_attentions value used at every step; optional final max_attentions /
 * alignments as the last sess.run would return them. */
int dctts_text2mel_generate(dctts_handle h, const int32_t* L, int32_t B, int32_t steps,
                            float* Y, int32_t* prev_hist,
                            int64_t* max_attentions, float* alignments, void* stream);
/* dctts_text2mel_generate with an end for each utterance.  Utterance b ends at
 *   len[b] = min(steps, j* + 1 + tail),  j* = the first frame whose attention argmax reaches stop_pos[b],
 * or at `steps` when no frame does (or stop_pos[b] < 0).  stop_pos and lengths (B) int32 are device pointers; tail >= 0.
 * Y rows < len[b] and prev_hist rows < len[b] are those of dctts_text2mel_generate on the same batch, bit for bit; Y rows
 * >= len[b] are 0 and prev_hist rows >= len[b] are -1 (prev_hist may be NULL).  On the persistent decode path a cluster
 * of utterances stops once all of them have ended (dctts_get_option "decode_last_frames": frames executed, summed over
 * clusters); the graph-per-frame loop (decode_mode 0) runs every frame and then applies the same rule. */
int dctts_text2mel_generate_until(dctts_handle h, const int32_t* L, int32_t B, int32_t steps,
                                  const int32_t* stop_pos, int32_t tail, float* Y, int32_t* prev_hist,
                                  int32_t* lengths, void* stream);
/* The autoregressive loop along a caller's attention windows: frame j of utterance b runs under the window path[b, j]
 * where synthesize.py:48 feeds prev_max_attentions = path[:, j] (path[b, 0] plays the role of the initial zeros) instead
 * of the previous frame's argmax.  path (B, steps) and lengths (B) int32 are device pointers; 1 <= steps <= max_T,
 * 1 <= lengths[b] <= steps, and 0 <= path[b, j] < max_N for j < lengths[b] -- anything else is refused before any launch
 * with a message that names the utterance (both arrays are read on the host).  Y rows < lengths[b] are what the
 * step-wise loop fed those windows computes; prev_hist (B,max_T) receives the path; optional argmax_hist (B,max_T) the
 * model's own argmax of each frame inside its forced window (where it would have moved).  Rows >= lengths[b] are 0 in Y
 * and -1 in prev_hist and argmax_hist.  A persistent decode cluster executes its longest length
 * ("decode_last_frames"); the graph-per-frame loop (decode_mode 0) runs `steps` frames. */
int dctts_text2mel_generate_path(dctts_handle h, const int32_t* L, int32_t B, int32_t steps, const int32_t* path,
                                 const int32_t* lengths, float* Y, int32_t* prev_hist, int32_t* argmax_hist,
                                 void* stream);
/* The same with path (B, steps) and lengths (B) in HOST memory.  Reading device arrays back makes
 * dctts_text2mel_generate_path wait for the stream; this form does not, so a caller that holds the path on the host can
 * queue one decode while the previous one runs.  The arrays may be reused as soon as the call returns. */
int dctts_text2mel_generate_path_host(dctts_handle h, const int32_t* L, int32_t B, int32_t steps,
                                      const int32_t* path_host, const int32_t* lengths_host, float* Y,
                                      int32_t* prev_hist, int32_t* argmax_hist, void* stream);
/* ---- aligning recorded speech to its text (DESIGN.md section 4d) ------------------ */
/* The best monotonic path through alignments (B, N, T) DEVICE float32 (e.g. dctts_train_eval's or
 * dctts_text2mel_align's): for utterance b with T_b = lengths_host[b] frames and text end e_b = ends_host[b] (its EOS
 * position), one character n_t per frame t < T_b with 0 <= n_0 <= w - 1, 0 <= n_t - n_{t-1} <= w - 1 and
 * n_{T_b - 1} = e_b (w = attention_win_size) -- the paths the decode can follow -- maximising the sum of
 * log(max(A[b, n_t, t], 1e-30f)) in float64; of two equal predecessors the smaller step wins.  Outputs, all DEVICE:
 * chars (B, T) int32 = n_t; path (B, T) int32 = the window of each frame, path[b, 0] = 0 and path[b, t] = n_{t-1}, as
 * dctts_text2mel_generate_path takes it; rows >= T_b are -1 in both; durations (B, N) int32 = frames per text position
 * (0 for a position the path steps over; they sum to T_b); score (B) float64 = the path's summed log-attention.
 * Refused before any launch, naming the utterance: T_b outside [1, T], e_b < 0 (the text has no EOS), e_b >= N,
 * e_b > (w - 1) T_b (the text is too long for the recording), or 2 (e_b + 1) doubles beyond the device's shared memory
 * per block.  The lengths and ends are read on the host; the search is one launch for the batch, with no host
 * synchronisation. */
int dctts_align_search(dctts_handle h, const float* alignments, int32_t B, int32_t N, int32_t T,
                       const int32_t* lengths_host, const int32_t* ends_host,
                       int32_t* path, int32_t* chars, int32_t* durations, double* score, void* stream);
/* The teacher-forced Text2Mel front and the search: L (B, max_N), mels (B, T, n_mels) DEVICE, 1 <= T <= max_T.  The
 * alignments are the dense softmax over all max_N keys of each frame's query, with AudioEnc fed the mels shifted by one
 * frame (train.py:51 at dropout 0); optional alignments (B, max_N, T) DEVICE receives them.  Then dctts_align_search with
 * N = max_N, with the same checks made before anything is launched.  Rows of mels at or past lengths_host[b] must be
 * zeros (as dctts_load_spectrograms_batch writes them): on the wgmma kernel set utterance b's outputs are then bit for
 * bit those of the call on that utterance alone at T = lengths_host[b]; on the fp32 set they agree within float32
 * rounding.  A trained handle with stale packing runs the fp32 kernels.  Clears the decode state that
 * dctts_decode_history reads. */
int dctts_text2mel_align(dctts_handle h, const int32_t* L, const float* mels, int32_t B, int32_t T,
                         const int32_t* lengths_host, const int32_t* ends_host,
                         int32_t* path, int32_t* chars, int32_t* durations, double* score,
                         float* alignments, void* stream);
/* ---- held-out quality: mel-cepstral distortion along a DTW alignment (DESIGN.md section 8h) ------------------ */
/* MCD-DTW between pairs of dB-normalised mel sequences (what Text2Mel produces and dctts_load_spectrograms_batch writes):
 * X (B, Tx, n_mels) and Y (B, Ty, n_mels) DEVICE float32; pair b compares X[b, :nx_host[b]] with Y[b, :ny_host[b]].
 * Per frame, in float64: a_m = (ln 10 / 20) (max_db x_m - max_db + ref_db) (the log amplitude, max_db and ref_db from
 * dctts_set_vocoder_params), c_k = sum_m a_m D[k, m] for k = 1 .. K, D the orthonormal DCT-II matrix
 * (D[k, m] = sqrt(2 / n_mels) cos(pi k (2m + 1) / (2 n_mels)); c_0, the energy, is left out).  Local cost
 * d(i, j) = (10 / ln 10) sqrt(2 sum_k (cx_ik - cy_jk)^2); D(0, 0) = d(0, 0), D(i, j) = d(i, j) + min(D(i-1, j-1),
 * D(i-1, j), D(i, j-1)), a tie going to the first of the three in that order (diagonal, advance X, advance Y); the
 * path ends at (nx_b - 1, ny_b - 1).  Outputs, DEVICE: mcd (B) float64 = D(nx_b - 1, ny_b - 1) / P_b with P_b the
 * cells on the path; pairs (B) int32 = P_b; path (B, Tx + Ty - 1, 2) int32 (i, j) from (0, 0), -1 past P_b, or NULL.
 * This is an MFCC-style distortion (a DCT of log mel amplitudes), not an SPTK / WORLD mel-cepstrum: its values are not
 * comparable to published MCD figures.  Refused before any launch, naming the utterance: nx_b outside [1, Tx], ny_b
 * outside [1, Ty], or three diagonals of nx_b doubles beyond the device's shared memory per block; K outside
 * [1, n_mels - 1].  Each pair's result does not depend on the other pairs.  One launch for the batch, with no host
 * synchronisation except the upload of D at the handle's first call; needs no parameters and leaves the decode and
 * training state alone. */
int dctts_mcd_dtw(dctts_handle h, const float* X, int32_t Tx, const int32_t* nx_host,
                  const float* Y, int32_t Ty, const int32_t* ny_host, int32_t B, int32_t K,
                  double* mcd, int32_t* pairs, int32_t* path, void* stream);
/* The long-form join (dc_tts_b200/longform.py): the decoded pieces of K texts into one mel sequence per text.
 * Y (P, T, n_mels) DEVICE, the pieces as dctts_text2mel_generate_until wrote them; piece_len (P) int32 DEVICE, their
 * lengths (clamped to [0, T]); piece_text_host (P) and piece_pause_host (P) HOST: each piece's text, 0 .. K-1 with every
 * text's pieces consecutive and in order, and the rows of `silence` that follow it (>= 0; 0 after a text's last piece).
 * out (K, T_out, n_mels) DEVICE: text k's pieces' rows < len in order, each but the last followed by its pause rows, then
 * zeros up to T_out; out_len (K) int32 DEVICE: each text's rows.  T_out must hold every text at full-length pieces
 * (sum over its pieces of T + pause), checked on the host with the other arguments before anything is launched.  One
 * launch; the offsets are a prefix sum of the device lengths inside the kernel, so the call does not wait for the decode
 * (only for the previous upload out of the handle's pinned staging buffer, as dctts_text2mel_generate_path_host). */
int dctts_join_rows(dctts_handle h, const float* Y, int32_t P, int32_t T, const int32_t* piece_len,
                    const int32_t* piece_text_host, const int32_t* piece_pause_host, int32_t K, float silence, int32_t T_out,
                    float* out, int32_t* out_len, void* stream);
/* synthesize.py:45-57 end to end with HOST buffers: copies L_host in, runs
 * dctts_text2mel_generate + dctts_ssrn, copies Y_host (B,max_T,n_mels; may be NULL) and
 * Z_host (B,4*max_T,F) out, and synchronises.  Host buffers should be pinned for speed. */
int dctts_synthesize_host(dctts_handle h, const int32_t* L_host, int32_t B,
                          float* Y_host, float* Z_host);

/* ---- vocoder ("next" row after the path: reference utils.py:67-114) --------------------- */
/* Signal-processing constants of hyperparams.py:13-24 (defaults = the LJ values: hop 275, win 1102, power 1.5,
 * max_db 100, ref_db 20, preemphasis 0.97, n_iter 50; n_fft = 2*(F-1) of the handle: 1024, 2048 or 4096, and
 * win_length <= n_fft, else the call fails).  preemphasis is float64:
 * the de-pre-emphasis filter runs with it as scipy.signal.lfilter does; the features' pre-emphasis rounds it to float32
 * as numpy does for a float32 waveform. */
int dctts_set_vocoder_params(dctts_handle h, int32_t hop_length, int32_t win_length, float power, float max_db,
                             float ref_db, double preemphasis, int32_t n_iter);
/* spectrogram2wav (utils.py:67-94) for a batch, entirely on the device: mag (B, T, F) normalised linear
 * magnitudes -> de-normalise, ^power, Griffin-Lim (n_iter x istft/stft with librosa's conventions), de-pre-emphasis.
 * wav (B, hop*(T-1)) DEVICE float32 receives the UNTRIMMED waveform; trim_host (B, 2) HOST int32 receives the
 * [start, end) sample range librosa.effects.trim (top_db 60) would keep.  n_iter < 0 means the configured value.
 * Synchronises `stream` before returning (trim_host is written by the host).  This is dctts_spectrogram2wav_momentum
 * with lengths_host NULL and momentum 0. */
int dctts_spectrogram2wav(dctts_handle h, const float* mag, int32_t B, int32_t T, int32_t n_iter, float* wav,
                          int32_t* trim_host, void* stream);
/* dctts_spectrogram2wav with a frame count per utterance, in one call at T.  lengths_host: (B) HOST int32 magnitude
 * frames, 2 <= lengths_host[b] <= T; a count outside that range fails the call, naming the utterance, before any
 * launch.  For each b, wav[b, :hop (T_b - 1)] and trim_host[b] are those of dctts_spectrogram2wav on mag[b:b+1, :T_b]
 * alone, bit for bit; wav[b] past that is 0.  Mag rows >= T_b are never read.  Synchronises `stream`.  This is
 * dctts_spectrogram2wav_momentum with momentum 0 (lengths_host is required here). */
int dctts_spectrogram2wav_ragged(dctts_handle h, const float* mag, int32_t B, int32_t T, const int32_t* lengths_host,
                                 int32_t n_iter, float* wav, int32_t* trim_host, void* stream);
/* dctts_spectrogram2wav / _ragged with the fast Griffin-Lim update (Perraudin, Balazs and Sondergaard 2013; librosa's
 * griffinlim(momentum=...)) and an optional per-iteration spectral convergence.  With alpha = momentum / (1 + momentum)
 * (float64, rounded to float32) and est_i = stft(istft(X_i)), est_{-1} = 0: c = est_i - alpha est_{i-1},
 * X_{i+1} = S c / max(1e-8, |c|); zero initial phase.  momentum must be finite and >= 0, else the call fails with a
 * message.  lengths_host: NULL, or (B) HOST frame counts as for dctts_spectrogram2wav_ragged.  convergence: NULL, or
 * (B, n_iter + 1) DEVICE float64 receiving ||S - |est_i||| / ||S|| over each utterance's frames, entry n_iter from one
 * more STFT of the final waveform (before de-emphasis).  At momentum 0 the waveform and trims equal
 * dctts_spectrogram2wav (lengths_host NULL) or dctts_spectrogram2wav_ragged, bit for bit, with or without convergence.
 * Synchronises `stream`. */
int dctts_spectrogram2wav_momentum(dctts_handle h, const float* mag, int32_t B, int32_t T, const int32_t* lengths_host,
                                   int32_t n_iter, double momentum, float* wav, int32_t* trim_host, double* convergence,
                                   void* stream);

/* Streaming Griffin-Lim (DESIGN.md section 8i): magnitude frames arrive in pieces, and each piece returns the samples
 * that are final.  For each utterance with A frames received, a push runs dctts_spectrogram2wav_momentum's iterations on
 * the prefix of A frames, with the samples already returned held at their values and only the frames that reach past
 * them taking part (warm-started from the previous push); it then returns the samples up to a look-ahead margin before
 * the prefix's end, or all of them once the utterance is final, de-emphasised from the float64 state the last push left.
 * A stream owns its buffers and tables (sized at open for T_cap frames per utterance), takes the vocoder parameters of
 * dctts_set_vocoder_params at open, and runs every launch on `stream`; close each stream before destroying its handle.
 * Errors are reported by dctts_last_error(h). */
typedef struct dctts_vocoder_stream_s* dctts_vocoder_stream;
/* B utterances of at most T_cap >= 2 frames each; n_iter < 0 means the configured value; momentum as for
 * dctts_spectrogram2wav_momentum.  *out receives the stream. */
int dctts_vocoder_stream_open(dctts_handle h, int32_t B, int32_t T_cap, int32_t n_iter, double momentum, void* stream,
                              dctts_vocoder_stream* out);
/* Appends rows_host[b] frames of mag (B, R, F) DEVICE float32 (row j of utterance b is its next frame j, j < rows_host[b] <= R)
 * and marks utterance b final where final_host[b] != 0 (final_host may be NULL: none).  One step runs for each utterance
 * that received rows or became final and has at least 2 frames.  counts_host (B) HOST receives the samples it committed,
 * and wav (B, ld) DEVICE float32 row b receives them, from its start; a count above ld fails the call before any launch.
 * Fails, naming the utterance, when rows arrive for an utterance after its final push, when T_cap would be exceeded, or
 * when a final utterance has fewer than 2 frames.  The returned samples concatenate, per utterance, to one waveform of
 * hop (T_b - 1) samples, untrimmed; with a single final push it is dctts_spectrogram2wav_momentum's with
 * lengths_host, bit for bit.  Asynchronous: the counts are known on the host, wav is written on `stream`. */
int dctts_vocoder_stream_push(dctts_vocoder_stream vs, const float* mag, int32_t R, const int32_t* rows_host,
                              const int32_t* final_host, float* wav, int64_t ld, int32_t* counts_host);
/* trim_host: NULL, or (B, 2) HOST int32 receiving the [start, end) librosa.effects.trim keeps of each streamed waveform
 * (every utterance must then be final).  Frees the stream whether or not the trims could be formed; synchronises `stream`. */
int dctts_vocoder_stream_close(dctts_vocoder_stream vs, int32_t* trim_host);

/* Streaming synthesis from text (DESIGN.md section 8j): the until-EOS decode publishes its progress to the host, SSRN runs
 * over windows of the published mel frames with the halo it needs, and a dctts_vocoder_stream turns them into samples while
 * the decode is still running.  Utterance b's mel frames are committed on a fixed grid of `chunk` frames (the last chunk
 * ends at its length); each chunk is one SSRN window and one vocoder push, in order, so the samples depend on the texts,
 * the weights and `chunk` alone, not on when the host polls.  Committed magnitude rows equal dctts_ssrn_ragged's on the
 * decode's Y bit for bit when the utterance's Y abs-max lies in [0.5, 1) (the windows' input planes use that fixed scale,
 * 2^15).  One stream per handle; while it is open, every entry point that writes the decode workspace or the weights or
 * grows a buffer (dctts_textenc, the generations, the teacher-forced graph, dctts_ssrn past max_T, dctts_reserve*, training, commit,
 * refresh) fails naming the open stream.  dctts_destroy closes an open stream (waiting for its decode).
 * Errors are reported by dctts_last_error(h). */
typedef struct dctts_synth_stream_s* dctts_synth_stream;
/* The mel frames of context SSRN needs before (*left) and after (*right) a run of committed frames, derived from the
 * committed layer table. */
int dctts_ssrn_halo(dctts_handle h, int32_t* left, int32_t* right);
/* Test aid: the stream's windowed SSRN on a caller's Y (B, T, n_mels) DEVICE.  Window b commits mel rows
 * [starts_host[b], starts_host[b] + counts_host[b]) of utterance b of length lengths_host[b] (1 .. T), reading rows
 * [max(0, start - left), min(length, end + right)); Z (B, 4 ldz_frames, F) DEVICE row b receives its 4 counts_host[b]
 * sigmoid rows from its start.  Synchronises `stream`. */
int dctts_ssrn_windows(dctts_handle h, const float* Y, int32_t B, int32_t T, const int32_t* starts_host, const int32_t* counts_host,
                       const int32_t* lengths_host, float* Z, int32_t ldz_frames, void* stream);
/* Opens a stream for B utterances of texts L (B, max_N) DEVICE int32, with dctts_text2mel_generate_until's stop positions
 * (stop_pos_host, HOST) and tail, `chunk` >= 1 mel frames per commit, and dctts_vocoder_stream_open's n_iter and momentum.
 * Allocates everything the stream needs, runs TextEnc and launches the decode on `stream`, and returns without waiting.
 * The decode takes the fewest utterances per cluster that leave one co-resident 16-CTA cluster slot free for the SSRN
 * and vocoder launches, where five per cluster allow it.  Fails without the persistent decode (after training:
 * dctts_refresh_synthesis), without a tensor-core SSRN chain, with chunk < 1, or when a stream is already open. */
int dctts_synth_stream_open(dctts_handle h, const int32_t* L, int32_t B, const int32_t* stop_pos_host, int32_t tail, int32_t chunk,
                            int32_t n_iter, double momentum, void* stream, dctts_synth_stream* out);
/* Runs every chunk that is ready (one SSRN launch set and one vocoder push per round, on the stream's own side stream) and
 * returns each utterance's newly committed samples, de-emphasised and untrimmed as dctts_vocoder_stream_push returns them:
 * wav (B, ld) HOST row b receives counts_host[b] samples, ld >= hop (4 max_T - 1); done_host[b] != 0 once utterance b
 * has had its last chunk; frames_host (B, HOST, or NULL) the mel frames utterance b's decode cluster had published when
 * the poll returned (never decreasing).  With `wait`, first blocks until a chunk is ready or every utterance is done,
 * failing with the decode's error if it failed.  Never synchronises the device. */
int dctts_synth_stream_poll(dctts_synth_stream ss, int32_t wait, float* wav, int64_t ld, int32_t* counts_host,
                            int32_t* done_host, int32_t* frames_host);
/* Waits for the decode, runs the remaining chunks, and frees the stream.  Outputs (each may be NULL; with all NULL the
 * stream is freed without running the rest): lengths_host (B) as dctts_text2mel_generate_until reports them; trim_host
 * (B, 2) as dctts_vocoder_stream_close; Y (B, max_T, n_mels) DEVICE the decode's mels, rows past each length 0; Z
 * (B, 4 max_T, F) DEVICE the committed magnitudes, rows past each length 0; first_frames_host (B) the frames the
 * utterance's decode cluster had published when its first chunk was pushed. */
int dctts_synth_stream_close(dctts_synth_stream ss, int32_t* lengths_host, int32_t* trim_host, float* Y, float* Z,
                             int32_t* first_frames_host);

/* Feature extraction (next row, SURVEY 8f-4): get_spectrograms -- utils.py:20-65 -- for ONE utterance from the
 * loaded waveform on: trim (librosa.effects.trim), pre-emphasis, STFT, |.|, mel filterbank
 * (librosa.filters.mel(sample_rate, n_fft, n_mels)), 20 log10, normalisation with the constants of
 * dctts_set_vocoder_params.  `wav` DEVICE float32 [n_samples]; `mel` (t_capacity, n_mels) and `mag`
 * (t_capacity, 1 + n_fft/2) DEVICE outputs, rows [0, *t_out) written, t_capacity >= 1 + n_samples / hop_length;
 * `trim_host` (optional) receives the [start, end) sample range kept.  Synchronises the stream once.
 * This is dctts_load_spectrograms_batch at B = 1 without the reduction (every frame is a mel row) and without padding:
 * the same two kernels compute it. */
int dctts_get_spectrograms(dctts_handle h, const float* wav, int64_t n_samples, int32_t sample_rate, float* mel, float* mag,
                           int32_t t_capacity, int32_t* t_out, int32_t* trim_host, void* stream);
/* load_spectrograms (utils.py:147-162) for B utterances at once, padded as one bucketed batch (data_load.py:122-129,
 * dynamic_pad).  wav: DEVICE, the B waveforms back to back; offsets_host: B+1 HOST int64 sample offsets;
 * dtype 0 = float32, 1 = int16 PCM (value / 32768, what utils._load_wav returns for int16 files).
 * Outputs are packed at the batch's own shape from the start of the caller's buffers (which hold t_capacity reduced
 * rows per utterance):  mel (B, T_b, n_mels) = every r-th frame,  mag (B, r*T_b, F);  rows past an utterance's own
 * length are zero.  t_host (B): reduced rows per utterance; trim_host (2B): [start, end) kept; *T_b_out = max t_host.
 * Each utterance's rows are bit for bit what dctts_get_spectrograms computes for it alone, then padded and reduced.
 * Two kernels per call whatever B is (trim energies of every utterance, then one CTA per STFT frame of the flattened
 * batch).  Fails, naming the utterance and writing nothing to mel or mag, when an utterance has fewer than 2 samples
 * left after trimming or T_b > t_capacity.  Synchronises once. */
int dctts_load_spectrograms_batch(dctts_handle h, const void* wav, int32_t dtype, const int64_t* offsets_host, int32_t B,
                                  int32_t sample_rate, float* mel, float* mag, int32_t t_capacity,
                                  int32_t* t_host, int32_t* trim_host, int32_t* T_b_out, void* stream);
/* What librosa.load(fpath, sr=sr_out) adds after decoding, for B utterances packed back to back: librosa 0.6
 * core.resample(y, sr_host[b], sr_out, res_type='kaiser_best', fix=True) = resampy 0.2 resample / resample_f.
 * wav: DEVICE, dtype 0 = float32, 1 = int16 PCM (value / 32768); offsets_host: B+1 HOST int64 sample offsets;
 * sr_host: B HOST native rates.  out: DEVICE float32, the B results back to back, at most out_capacity samples;
 * out_offsets_host (B+1) receives their offsets.  Per utterance, with ratio = float(sr_out) / sr_in:
 *   - sr_in == sr_out: returned unchanged (librosa's early return), only converted to float32;
 *   - otherwise int(n ratio) samples of resample_f, zero-padded to ceil(n ratio) (util.fix_length).  Output t:
 *     n = int(reg), frac = scale (reg - n), scale = min(1, ratio), offset = int(512 frac), eta = 512 frac - offset;
 *     left wing i < min(n + 1, (nwin - offset) // index_step) on x[n - i], then frac = scale - frac and the right wing
 *     k < min(n_in - n - 1, (nwin - offset) // index_step) on x[n + k + 1], weight win[j] + eta delta[j] at
 *     j = offset + i index_step, index_step = int(512 scale); a float32 accumulator, each tap rounded
 *     float32(double(y) + weight double(x)).  reg is the float64 register resampy advances by 1 / ratio per output.
 *   - the filter is kaiser_best: the half window rolloff sinc(rolloff linspace(0, 64, 64*512 + 1)) times the right half
 *     of a Kaiser window (beta 14.769656459379492, rolloff 0.9475937167399596), times ratio when ratio < 1; delta is its
 *     first difference, 0 at the end.
 * One kernel, no synchronisation: a following dctts_load_spectrograms_batch(dtype = 0) on the same stream keeps its one.
 * Fails, naming the utterance, with nothing written or launched, on a rate <= 0, an input of 0 samples, an output
 * shorter than 1 sample (int(n ratio) < 1, where resampy raises) or more than out_capacity samples in all. */
int dctts_resample_batch(dctts_handle h, const void* wav, int32_t dtype, const int64_t* offsets_host, const int32_t* sr_host,
                         int32_t B, int32_t sr_out, float* out, int64_t out_capacity, int64_t* out_offsets_host, void* stream);
/* The time register dctts_resample_batch computes for n_out outputs from sr_in to sr_out, as the affine segments the
 * kernel evaluates: register(t) = v0[i] + (t - t0[i]) step[i] for t0[i] <= t < t0[i+1].  Returns the number of
 * segments, or -1 for bad arguments or more than `capacity`.  No handle, no GPU. */
int32_t dctts_resample_time_register(int64_t n_out, int32_t sr_in, int32_t sr_out, int64_t* t0, double* v0, double* step,
                                     int32_t capacity);

/* ---- training step (BASELINE config 5; SURVEY 8f-3) --------------------------------------
 * One optimiser step of the reference's Text2Mel trainer -- graph train.py:43-68 in mode "train" (dropout after
 * every block, full softmax attention), losses train.py:83-99 (L1 + sigmoid cross-entropy on the mels + guided
 * attention), elementwise clipping to [-1, 1] and tf.train.AdamOptimizer defaults with the Noam learning rate
 * (train.py:122-132, utils.py:141-145) -- for fixed-size batches L (B, max_N) int32, mels (B, max_T, n_mels), DEVICE
 * pointers.  All tensors are float32; the three GEMMs of every block (forward conv, data gradient, weight gradient) run on
 * wgmma as split-fp16 x3 with per-tensor power-of-two scales (option "train_tc", default 7; 0 = the float32 CUDA-core
 * kernels).  dctts_train_init allocates the saved activations and the gradient / Adam arenas and switches the handle's
 * SYNTHESIS entry points to the fp32 kernel set (the optimiser updates the fp32 weights only, the packed planes go stale;
 * dctts_refresh_synthesis packs them again).
 * Dropout uses a stateless hash of (element, block index, seed) -- TF's random stream cannot be reproduced.
 * losses_host (optional): {total, mels L1, binary divergence, guided attention}; reading them synchronises.
 * apply = 0 leaves the gradients in the arena (dctts_train_grads: one flat device buffer, what a data-parallel job
 * all-reduces) for dctts_train_apply.  dctts_train_tensor copies a variable (what = 0), its gradient (1) or Adam
 * moments (2, 3) to the host, in the TF variable's own layout. */
int dctts_train_init(dctts_handle h, int32_t B, float dropout_rate);
int dctts_train_step(dctts_handle h, const int32_t* L, const float* mels, int32_t B, int64_t global_step, uint32_t seed, float lr,
                     int32_t apply, float* losses_host, void* stream);
/* The same step on a length-bucketed batch at its own shape (the reference's dynamic_pad=True, data_load.py:122-129):
 * L (B, N) int32 and mels (B, T, n_mels), packed at that shape.  Capacity: 1 <= N <= max_N and 1 <= T <= max_T of the
 * hparams the handle was created with, or more after dctts_train_reserve (texts longer than 180 need a handle with a
 * larger max_N or a reserve; any max_N >= 1 is accepted, and one too large for device
 * memory fails where its workspace is allocated); B must be
 * the batch size given to dctts_train_init.  A step outside the capacity fails with a message and launches nothing.
 * The losses are the reference's at this shape: means over B T n_mels; the guided-attention sum over the N x T corner of
 * the (max_N, max_T) weight table divided by B N T (train.py:91-95).  The softmax runs over the N keys and TextEnc's SAME
 * padding sees the edge of the tensor at N.  dctts_train_step is this call at (max_N, max_T).
 * Determinism: by default the weight, LayerNorm, bias and embedding gradients and the loss sums are added with float
 * atomics, so two identical steps may differ in the last bits.  With the option "train_deterministic" = 1 every sum runs in
 * a fixed order, and dctts_train_step(_shaped), dctts_train_step_ssrn(_shaped), dctts_train_apply and
 * dctts_train_eval(_ssrn) write the same bits -- variables, Adam m and v, the gradient arena, losses_host, and the
 * evaluations' Y, Z and alignments -- whenever they get the same variables, Adam moments, global step, batch (same shape),
 * seed, lr, dropout rate, batch size and "train_tc" kernel set, whatever the workspace capacity (dctts_train_reserve),
 * whatever ran on the handle before (evaluations, synthesis, dctts_refresh_synthesis, a step with apply = 0 followed by
 * dctts_train_apply) and on whichever handle.  No split count of this mode is read from the device.  Not promised: equal
 * bits between kernel sets, or with the default mode.  The mode's partial sums live in the training workspace (allocated
 * at its first step, kept across dctts_train_reserve). */
int dctts_train_step_shaped(dctts_handle h, const int32_t* L, int32_t N, const float* mels, int32_t T, int32_t B, int64_t global_step,
                            uint32_t seed, float lr, int32_t apply, float* losses_host, void* stream);
int dctts_train_apply(dctts_handle h, int64_t global_step, float lr, void* stream);
/* A forward-only evaluation of the Text2Mel training graph on one batch: what the reference computes for
 * sess.run(g.alignments) or sess.run(g.merged) (train.py:100-104,156) -- the step's forward at (N, T) with its dropout mask at
 * `seed`, on the kernel set "train_tc" selects, and the step's losses at that shape into losses_host = {total, mels L1,
 * binary divergence, guided attention} (optional; reading them synchronises).  Y_out (B, T, n_mels) = sigmoid(logits) and
 * align_out (B, N, T), DEVICE pointers, are written when non-NULL.  It accepts exactly the shapes dctts_train_step_shaped
 * accepts and fails, before launching anything, with its message outside them.  It writes neither the variables, the
 * gradient arena (dctts_train_grads: an eval between a step with apply = 0 and dctts_train_apply leaves it as it was) nor
 * the Adam moments, so a step after an eval is the step without it. */
int dctts_train_eval(dctts_handle h, const int32_t* L, int32_t N, const float* mels, int32_t T, int32_t B, uint32_t seed,
                     float* Y_out, float* align_out, float* losses_host, void* stream);
/* The SSRN counterpart (train.py:115-118): Z_out (B, 4T, F) = sigmoid(logits), DEVICE, optional; losses_host = {total,
 * mags L1, binary divergence}; the shapes of dctts_train_step_ssrn_shaped; the same state contract. */
int dctts_train_eval_ssrn(dctts_handle h, const float* mels, const float* mags, int32_t B, int32_t T, uint32_t seed, float* Z_out,
                          float* losses_host, void* stream);
/* The SSRN trainer (train.py num = 2: SSRN on the GROUND-TRUTH mels :69-72, losses :100-108, same optimiser): mels
 * (B, T, n_mels), mags (B, 4T, 1 + n_fft/2) DEVICE pointers; losses_host = {total, mags L1, binary divergence, 0}.
 * A handle trains one of the two networks at a time (the init call selects which).  The T given to dctts_train_init_ssrn
 * is a capacity: dctts_train_step_ssrn_shaped steps at any 1 <= T <= capacity (means over B 4T F), keeping the Adam state;
 * a step beyond it fails with a message and launches nothing.  dctts_train_step_ssrn is this call at the capacity. */
int dctts_train_init_ssrn(dctts_handle h, int32_t B, int32_t T, float dropout_rate);
int dctts_train_step_ssrn(dctts_handle h, const float* mels, const float* mags, int32_t B, int64_t global_step, uint32_t seed, float lr,
                          int32_t apply, float* losses_host, void* stream);
int dctts_train_step_ssrn_shaped(dctts_handle h, const float* mels, const float* mags, int32_t B, int32_t T, int64_t global_step,
                                 uint32_t seed, float lr, int32_t apply, float* losses_host, void* stream);
/* Grow the training workspace of the network being trained (the last init call's) to at least N text positions (Text2Mel;
 * ignored for SSRN) and T mel frames, so that the shaped steps accept 1 <= N <= N_cap and 1 <= T <= T_cap.  Without a
 * reserve call the capacity is the init call's: (max_N, max_T) for Text2Mel, T for SSRN.  Never shrinks; a no-op when the
 * workspace already fits; otherwise it synchronises the device and re-allocates only the shape-dependent buffers: the
 * variables, the gradient arena (and its address, dctts_train_grads) and the Adam moments are kept, so training continues
 * where it was.  The guided-attention table stays (max_N, max_T): a Text2Mel step past it takes the guided-attention loss
 * over the min(N, max_N) x min(T, max_T) corner divided by B min(N, max_N) min(T, max_T) (train.py:91-95 pads with -1 and
 * crops to the table), and keys or frames outside that corner get the mel losses' gradients only.  A failed growth (out of
 * memory) leaves the old capacity.  dctts_train_capacity reports (N_cap, T_cap); N_cap is 0 for SSRN. */
int dctts_train_reserve(dctts_handle h, int32_t N, int32_t T);
int dctts_train_capacity(dctts_handle h, int32_t* N, int32_t* T);
int dctts_train_grads(dctts_handle h, float** grads, int64_t* count);
int dctts_train_tensor(dctts_handle h, const char* tf_name, int32_t what, float* host_out, int64_t count);
/* Inverse of dctts_train_tensor for what = 0 (variable), 2 (Adam m), 3 (Adam v): restores a training state (resume). */
int dctts_train_set_tensor(dctts_handle h, const char* tf_name, int32_t what, const float* host_in, int64_t count);
/* Synthesis from the variables being trained.  Every call that writes a variable -- dctts_train_init, a step with apply = 1,
 * dctts_train_apply, dctts_train_set_tensor with what = 0 -- leaves the handle's packed weights stale: synthesis runs on the
 * fp32 kernel set with the graph-per-frame decode, and dctts_set_tensor_path(1) fails.  This call packs the wgmma weight
 * planes, the persistent decode's weight stream and its LayerNorm parameters again on the device from the variables as
 * they are, so that afterwards the handle selects its kernels and computes exactly what a freshly committed handle
 * holding the same variables would: tensor path 1, the persistent decode where it can be placed (the captured AR step is
 * dropped).  It writes none of the variables, the Adam moments, the gradient arena or the training workspace, and a step
 * with apply = 0 or an evaluation (dctts_train_eval*) keeps it in force.  A no-op on a handle whose packed weights are
 * current (one never trained, or refreshed since its last update).  Synchronises `stream` and the device; costs one
 * abs-max reduction, one small device-to-host copy and one pass over the weights. */
int dctts_refresh_synthesis(dctts_handle h, void* stream);

/* ---- utilities ----------------------------------------------------------------- */
/* Pre-size the workspace (otherwise grown lazily on first use) for batches up to B. */
int dctts_reserve(dctts_handle h, int32_t max_batch);
/* Grow the buffers the full-sequence chains run in so that dctts_ssrn / dctts_ssrn_ragged take B utterances of T mel
 * frames, T above max_T too, without allocating: r x B x T rows, 98688 bytes per frame at the LJ hyperparameters (c 512,
 * d 256, F 1025).  Only ever grows and keeps the weights; it synchronises the device when it grows.  The new buffers are
 * allocated before the old ones are freed: a size that cannot be allocated fails, naming the bytes, and leaves the
 * handle as it was.  bytes (optional) receives what those buffers hold after the call. */
int dctts_reserve_frames(dctts_handle h, int32_t B, int32_t T, int64_t* bytes);
/* Number of kernels this library has launched on the handle since creation (graph
 * replays count their kernel nodes). */
int64_t dctts_launch_count(dctts_handle h);
/* Host utility for the checkpoint reader (dc_tts_b200/checkpoint.py): CRC-32C (Castagnoli) of `n` bytes,
 * continuing from `crc` (0 to start) -- the checksum TF's tensor bundle stores (masked) for every index
 * block and every tensor restored at synthesize.py:31-41.  No handle, no GPU. */
uint32_t dctts_crc32c(uint32_t crc, const void* data, int64_t n);
/* Selects the kernel set: 0 = one fp32 CUDA-core GEMM + one LN kernel per block (baseline),
 * 1 = default: wgmma split-fp16 (3-MMA, fp32-grade) fused blocks where they apply (whole
 * networks, full-sequence attention, and the wide AudioDec rows of the graph decode step when B >= 8). */
int dctts_set_tensor_path(dctts_handle h, int32_t mode);

/* Kernel-variant switches (every value is a parity-tested code path; defaults = measured best):
 *   "decode_mode"  1 = the whole AR loop (synthesize.py:45-54) as ONE persistent cluster kernel (default),
 *                  0 = one captured CUDA graph per mel frame (round-1 path)
 *   "tc_occ2" 0/1, "tc_mcast" 0/1, "tc_resid_tma" 0/1: wgmma block kernel variants
 *   "fused_ln" 0/1: graph decode, GEMM + LN in one launch;  "tc_debug" 0/1;  "decode_prof" 0/1;  "pdl" 0/1 (process-wide)
 *   "decode_force_prepass" 0/1: measurement / test switch of the persistent decode (default 0): every utterance takes the
 *                  receptive-field recompute at every frame j >= 1, as if its attention window had moved (the worst case)
 *   "train_tc" 0..7: training GEMMs on wgmma, bit mask 1 forward conv (+ wgmma attention), 2 data gradient, 4 weight gradient
 *   "train_deterministic" 0/1 (default 0): the training step's sums in a fixed order, so that a seeded run repeats bit for
 *                  bit (see dctts_train_step_shaped); it may change between steps and does not affect synthesis
 *   "chain_history" 0/1 (default 0): test aid, the full-sequence chains keep every block's rows for dctts_chain_history
 *   "decode_group" 0..5 (default 0): measurement switch, utterances per persistent-decode cluster; 0 = the library's rule
 *                  (the fewest that keep every cluster co-resident; a synthesis stream's leaves one cluster slot free)
 *   "decode_timing" 0/1 (default 0): measurement switch, CUDA events around every persistent-decode launch; dctts_get_option
 *                  "decode_last_us" then gives the last launch's GPU time in microseconds (waits for it)
 * dctts_get_option also answers "decode_available" (1 when this handle / device can run the persistent decode),
 * "decode_max_clusters" (16-CTA clusters of the decode kernel that are co-resident on this device) and, once the
 * parameters are committed, "ssrn_tc_available" (1 when every SSRN block has a wgmma kernel, the F-wide ones included:
 * at F = 2049 they need a 16-CTA cluster; when none can be scheduled on the device the call fails and says so), and
 * "decode_last_frames": frames the last generation executed, summed over the persistent decode's clusters (the
 * graph-per-frame loop: its step count); synchronises the device. */
int dctts_set_option(dctts_handle h, const char* name, int32_t value);
int dctts_get_option(dctts_handle h, const char* name, int32_t* value);
/* Of the last dctts_text2mel_generate on the persistent decode path: frames in which a cluster had to recompute the
 * AudioDec receptive field because an attention window moved (summed over clusters), utterance-frames recomputed,
 * clusters launched.  Synchronises the device. */
int dctts_decode_stats(dctts_handle h, int32_t* moved_frames, int32_t* moved_utterance_frames, int32_t* clusters);
/* SM-clock lap timers (cycles) of the last persistent decode run with option "decode_prof" = 1: cluster 0, CTA rank 0.
 * n <= 24.  Buckets of thread 0, which together cover the kernel: 0 block start, 1 weight-stream wait, 2 GEMV, 3 slot release,
 * 4 all-gather, 5 cluster barrier, 6 LayerNorm, 7 mix, 8 attention, 9 recompute attention; the recompute GEMM as 10 waiting
 * for the block's weight chunks, 11 descriptor table, 12 issuing the A slabs, 13 draining the MMAs and epilogue stores,
 * 14 weight refill and LayerNorm parameters; 15 recompute LayerNorm, 16 recompute barriers, 17 frame bookkeeping;
 * 21 issuing the next block's parameter and tap prefetch.  In the one-row pass, 4 is finishing the slice and storing it
 * to every CTA, 5 waiting for the other CTAs' slices, 6 merging their LayerNorm statistics.
 * Buckets of the recompute's MMA warpgroup (thread 128), which overlap the above: 18 waiting for A slabs, 19 issuing the MMAs
 * and waiting for the slab before, 20 epilogue stores. */
int dctts_decode_profile(dctts_handle h, int64_t* cycles, int32_t n);
/* Test aid: the decode state of the last generation on the handle (dctts_text2mel_generate without max_attentions and
 * alignments, _generate_until, _generate_path, dctts_synthesize_host), copied into caller DEVICE memory, n elements, in the
 * order of the utterances the library decoded (the generation's B):
 *   what 0: AudioEnc block `layer`'s output rows (B, T, d)         what 3: K | V (B, N, 2d)
 *   what 1: AudioDec block `layer`'s output rows (B, T, d), the     what 4: Y (B, T, n_mels), rows past a length included
 *           last block's logits (B, T, n_mels)                      what 5: the window of every frame (B, T) int32
 *   what 2: R = [context | Q] (B, T, 2d)
 * with T = max_T, N = max_N.  A row holds what the decode last wrote there; which rows are current depends on the decode
 * (DESIGN.md, "The decode one block at a time").  The graph-per-frame decode (option decode_mode 0) on the tensor path at
 * B >= 8 keeps the outputs of the AudioDec blocks whose successor also runs on the tensor cores as split-fp16 planes only:
 * for those, the rows are hi + lo of the planes and *joined (optional) is set to 1, else 0.
 * Fails with a message, copying nothing, when the handle's last writer of these buffers was anything but such a generation
 * (a generation with the final attention pass, dctts_text2mel_forward, dctts_textenc, a workspace growth), or on a bad
 * `what`, `layer` or n.  Launches no kernel; synchronises `stream`. */
int dctts_decode_history(dctts_handle h, int32_t what, int32_t layer, void* out, int64_t n, int32_t* joined, void* stream);
/* Test aid (option chain_history = 1, default 0): the rows the last call's full-sequence chains left, copied into caller
 * DEVICE memory as float32, B * L rows of C, in the caller's order of the utterances.  net: 0 TextEnc, 1 AudioEnc, 2 AudioDec,
 * 3 SSRN, 4 the attention.  what 0: block `layer`'s output (the attention's layer 0 is R = [context | Q]); what 1 (layer 0):
 * the first block's input as its kernel read it.  Kept by dctts_textenc, _audioenc, _audiodec, _ssrn, _ssrn_ragged on the
 * tensor path, _text2mel_forward (TextEnc, AudioEnc, the attention, AudioDec) and _text2mel_align (the first three).
 * On the tensor path the hidden blocks' outputs and the first block's input are split-fp16 planes: the rows are then hi + lo,
 * times the utterance's inverse input scale for a scaled network input (exact: the scale is a power of two), and *joined
 * (optional) is set to 1, else 0.  dctts_chain_history_shape gives (B, L, C) of a record.
 * Fails with a message naming the reason, copying nothing, when the last call that ran synthesis kernels or changed the
 * weights did not run a full-sequence chain of `net` with the option on: a decode, an op-level block, embedding, LayerNorm
 * or attention call, the alignment search, MCD-DTW, a workspace growth, another network's chain, the option off,
 * dctts_synthesize_host, per-utterance lengths on the fp32 kernels (run once per utterance, not kept), a parameter commit,
 * a training update or dctts_train_set_tensor, dctts_refresh_synthesis; or when the caller did not ask for the rows (the
 * logits).  Calls that touch neither (the training forward and loss without an update, the training test aids, the
 * vocoder and feature extraction) leave the records readable.  Launches no kernel; synchronises `stream`.  With the option
 * off the chains copy nothing and launch the same kernels. */
int dctts_chain_history_shape(dctts_handle h, int32_t net, int32_t layer, int32_t what, int32_t* B, int32_t* L, int32_t* C);
int dctts_chain_history(dctts_handle h, int32_t net, int32_t layer, int32_t what, float* out, int64_t n, int32_t* joined,
                        void* stream);
/* Measurement aid for bench.py's roofline leg: runs the block `scope` on a synthetic
 * (B,L,Cin) input `warmup`+`iters` times and returns the mean device time of each of its
 * kernels (CUDA events on `stream` around every launch), ms_per_kernel[0..*n_kernels), <= 8. */
int dctts_bench_block(dctts_handle h, const char* scope, int32_t B, int32_t L, int32_t iters,
                      int32_t warmup, float* ms_per_kernel, int32_t* n_kernels, void* stream);
/* Test aid: ONE conv-GEMM of the training step on caller DEVICE tensors, through the launch functions the step calls;
 * the training state is not touched (the wgmma set gets a workspace and fresh abs-max slots of its own).
 *   impl 0: the float32 CUDA-core kernels (tiled conv GEMM, conv_wgrad_kernel); impl 1: the wgmma split-fp16 kernels.
 *   mode 0: out[b,t,n] (+)= bias[n] + sum_j sum_k X[b, t+shifts[j], k] W_j[k][n]   (zero outside [0, L) of utterance b)
 *           Wd = W_0 | W_1 | ... each [K][ldwd]; out (B, L, ldo) with ldo == ldwd; bias has ldwd floats; accumulate 0 or 1.
 *   mode 1: out_j[k][n] += sum_b sum_t X[b, t+shifts[j], k] dY[b,t,n]
 *           Wd = dY, B*L rows of pitch ldwd; out = out_0 | out_1 | ... each [K][ldo]; bias NULL, accumulate 1.
 * X: B*L rows of pitch ldx.  1 <= ntaps <= 3; shifts_host: ntaps HOST ints.  Fails with a message, leaving out untouched, when
 * a pitch is not a multiple of 4 or narrower than its width, a tensor is not 16-byte aligned, or (impl 1) the wgmma
 * kernels' preconditions do not hold: it never switches to the other kernel set.  Synchronises `stream`. */
int dctts_conv_gemm(dctts_handle h, int32_t impl, int32_t mode, const float* X, int32_t ldx, int32_t B, int32_t L, int32_t K,
                    const float* Wd, int32_t ldwd, int32_t N, int32_t ntaps, const int32_t* shifts_host, const float* bias,
                    int32_t accumulate, float* out, int32_t ldo, void* stream);
/* Test aid: the backward of ONE block's dropout / activation / highway gate / LayerNorm on caller DEVICE tensors, through the
 * launch function the training step calls (one launch); the training state is not touched.
 *   mode 0: conv1d or transposed conv, out = dropout(act(LN(pre[:, 0:C]; g1, b1))), act 0 none / 1 ReLU (mask z > 0);
 *   mode 1: highway, out = dropout(h1 h2 + (1 - h1) x), h1 = sigmoid(LN(pre[:, 0:C]; g1, b1)), h2 = LN(pre[:, C:2C]; g2, b2);
 *   LayerNorm: biased variance, eps 1e-12.  nconv = C (mode 0) or 2C (mode 1).
 * pre (rows, ldy >= nconv) the pre-LN conv output; gout (rows, ldg >= C) the gradient of out; X (rows, ldx >= C) the
 * block input (mode 1; NULL otherwise); ln (4, C) = g1 | b1 | g2 | b2 (g2, b2 unused in mode 0).  The dropout mask is the
 * step's: element (row, c) is kept iff its hash of (row C + c, layer, seed) clears dropout_rate, kept values scaled by
 * 1 / (1 - dropout_rate); rate 0 keeps everything.
 * Out: dy (rows, ldy) the gradient of pre (columns [0, nconv)); gin (rows, ldg, mode 1) the highway part g (1 - h1) of the
 * input gradient; dparams (4C + nconv) floats ADDED onto: dg1 | db1 | dg2 | db2 | dbias (dg2, db2 untouched in mode 0).
 * Pad columns are neither read nor written.  Fails with a message, launching nothing, on a bad mode, act, rate or pitch,
 * a highway block wider than 1056 channels or any block wider than 2080.  Synchronises `stream`. */
int dctts_block_bwd(dctts_handle h, int32_t mode, int32_t act, int64_t rows, int32_t C, const float* pre, int32_t ldy,
                    const float* gout, int32_t ldg, const float* X, int32_t ldx, const float* ln, float dropout_rate, int32_t layer,
                    uint32_t seed, float* dy, float* gin, float* dparams, void* stream);
/* Test aid: the forward twin of dctts_block_bwd, the LayerNorm epilogue of the training forward on caller DEVICE tensors,
 * through the launch the step makes (launch_ln_rows with the step's dropout mask):
 *   mode 0: out = dropout(act(LN(pre[:, 0:C]; g1, b1)));  mode 1: out = dropout(h1 h2 + (1 - h1) x), as dctts_block_bwd.
 * pre (rows, ldy), X (rows, ldx, mode 1), ln (4, C), the mask of (row C + c, layer, seed) as dctts_block_bwd's; out (rows,
 * ldo >= C), pad columns untouched.  Fails with a message, launching nothing, on a bad mode, act, rate or pitch, or a width
 * past the widest LayerNorm kernel (2080).  Synchronises `stream`. */
int dctts_block_fwd(dctts_handle h, int32_t mode, int32_t act, int64_t rows, int32_t C, const float* pre, int32_t ldy,
                    const float* X, int32_t ldx, const float* ln, float dropout_rate, int32_t layer, uint32_t seed, float* out,
                    int32_t ldo, void* stream);
/* Test aid: the attention backward of the Text2Mel training step (three launches: guided-attention sum, query side, key side)
 * on caller DEVICE tensors, through the launch function the step calls, with the handle's d (the kernels need d = 256).
 * gR (B,T,2d) the gradient of R = [ctx ; Q]; Q (B,T,d); KV (B,N,2d) = [K | V]; align (B,N,T) the forward's softmax over
 * n; gts the guided-attention weights, >= n_lim rows of stride ld_gts >= t_lim, of which the (n_lim, t_lim) corner is read.
 * With S = Q K^T / sqrt(d), A = align (used as given), loss = sum_corner |A gts| / (B n_lim t_lim):
 *   gQ (B,T,d) = gR[:, :, d:2d] + dS K / sqrt(d);  gKV (B,N,2d) = [dS^T Q / sqrt(d) | A dctx];  sums[2] += sum_corner |A gts|
 * with dA = dctx V^T + sign(A gts) gts / (B n_lim t_lim) inside the corner, dS = A (dA - sum_n A dA).  sums: 3 doubles, only
 * sums[2] is written.  The call owns the (B,T,N) dS scratch.  Fails with a message, launching nothing, when d != 256, the
 * crop does not fit (1 <= n_lim <= N, 1 <= t_lim <= T, t_lim <= ld_gts) or N keys need more shared memory than the device
 * allows.  Synchronises `stream`. */
int dctts_attn_bwd(dctts_handle h, const float* gR, const float* Q, const float* KV, const float* align, const float* gts,
                   int32_t ld_gts, int32_t B, int32_t T, int32_t N, int32_t n_lim, int32_t t_lim, float* gQ, float* gKV, double* sums,
                   void* stream);
/* Test aid: the mel / magnitude losses of the training step on caller DEVICE tensors, through the launch functions the step
 * calls.  logits (rows, ldl >= C), target (rows, C) dense, n = rows C, y = sigmoid(logits):
 *   sums[0] += sum |y - target|,  sums[1] += sum BCE(logits, target),  dlogits (rows, ldg >= C) = (sign(y - t) y (1 - y) + y - t) / n
 * and, when Y is not NULL, Y (rows, C) dense = y (a second launch, the one the training-graph evaluation makes).  Pad
 * columns are neither read nor written.  Fails with a message on a bad shape or pitch.  Synchronises `stream`. */
int dctts_train_loss(dctts_handle h, const float* logits, int32_t ldl, const float* target, int64_t rows, int32_t C, float* dlogits,
                     int32_t ldg, float* Y, double* sums, void* stream);
/* Test aid: ONE stage of dctts_spectrogram2wav on caller DEVICE tensors, through the launch functions the product calls,
 * with the handle's vocoder parameters and the tables (twiddles, window, window sum-square) it builds for (T, win, hop).
 * Ly = hop (T - 1), nfr = 1 + Ly / 512, F = 1 + n_fft / 2.
 *   0 prepare:    in = mag (B,T,F) float32            -> out = X (B,T,F) complex64  (S = Re X, zero phase)
 *   1 istft:      in = X (B,T,F) complex64            -> out = wav (B,Ly) float32
 *   2 stft_phase: in = wav (B,Ly), S (B,T,F) float32  -> out = X (B,T,F) complex64
 *   3 deemph:     in = out = wav (B,Ly), in place
 *   4 energies:   in = wav (B,Ly)                     -> out = mse (B,nfr) float32; trim_host (B,2) HOST int32 (optional)
 *                 receives the [start, end) ranges dctts_spectrogram2wav would report for this waveform.
 * Fails with a message on a bad stage or shape.  Synchronises `stream`. */
int dctts_vocoder_stage(dctts_handle h, int32_t stage, int32_t B, int32_t T, const void* in, const float* S, void* out,
                        int32_t* trim_host, void* stream);
/* Test aid: ONE stage of dctts_load_spectrograms_batch on caller DEVICE tensors, through the launch functions the product
 * calls, with the handle's vocoder parameters and the feature tables it builds for `sample_rate`.  wav: packed samples,
 * dtype 0 float32 or 1 int16 (value / 32768).  F = 1 + n_fft / 2.
 *   0 energies: seg_host = B + 1 HOST sample offsets of whole utterances -> out = mse float32, utterance b's 1 + n_b / 512
 *               frame energies (librosa.effects.trim's) back to back; host_out (B,2) HOST int32 receives the [start, end)
 *               ranges dctts_load_spectrograms_batch would keep.
 *   1 spectra:  seg_host = (B,2) HOST int64 (first sample, length >= 2) of already trimmed utterances, reduction r ->
 *               out = mag (B, r T_b, F), out2 = mel (B, T_b, n_mels) float32.  Utterance b's T = 1 + length / hop frames
 *               write mag rows t < T and mel rows t / r for t % r == 0 (T_b >= ceil(T / r)); no other element is written.
 *   2 tables:   out = the uploaded mel weights (n_mels, F) float32, out2 = the Hann window (win) float32, host_out
 *               (n_mels,2) HOST int32 = each filter's [first, last + 1) non-zero FFT bins.
 * Fails with a message on a bad stage, segment or T_b.  Synchronises `stream`. */
int dctts_feature_stage(dctts_handle h, int32_t stage, int32_t sample_rate, const void* wav, int32_t dtype, const int64_t* seg_host,
                        int32_t B, int32_t r, int32_t T_b, void* out, void* out2, int32_t* host_out, void* stream);
/* Test aid: ONE fast Griffin-Lim phase step of dctts_spectrogram2wav_momentum on caller DEVICE tensors, through the
 * same launch function, like dctts_vocoder_stage 2: in = wav (B,Ly) float32 and S (B,T,F) float32; E (B,T,F) complex64
 * holds est_{i-1} on entry and est_i on return; X (B,T,F) complex64 receives S c / max(1e-8, |c|).  partials: NULL, or
 * (B,T) float32 receiving each frame's sum_k (S - |est_i|)^2.  Always runs the momentum kernel (at momentum 0,
 * c = est_i - 0 est_{i-1}).  Fails with a message on a bad momentum.  Synchronises `stream`. */
int dctts_vocoder_momentum_step(dctts_handle h, int32_t B, int32_t T, const float* wav, const float* S, void* E, void* X,
                                double momentum, float* partials, void* stream);
/* Raw device memory helpers so that a host without torch can drive the library. */
int dctts_malloc(dctts_handle h, void** ptr, int64_t bytes);
int dctts_free(dctts_handle h, void* ptr);
int dctts_memcpy_h2d(dctts_handle h, void* dst, const void* src, int64_t bytes, void* stream);
int dctts_memcpy_d2h(dctts_handle h, void* dst, const void* src, int64_t bytes, void* stream);
int dctts_malloc_host(dctts_handle h, void** ptr, int64_t bytes);   /* pinned */
int dctts_free_host(dctts_handle h, void* ptr);
int dctts_stream_sync(dctts_handle h, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* DCTTS_H_ */
