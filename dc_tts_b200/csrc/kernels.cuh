// kernels.cuh -- argument blocks and launchers shared by the kernel files and the C-ABI.
//
// Row addressing (all kernels): an activation tensor is (B, L, C) float32 channels-last
// with leading dimension ld (floats).  A launch covers, for every batch element b, the
// time rows t in [t_end-R+1, t_end] where t_end = *jptr (device int, the AR step) when
// jptr != nullptr, else L-1.  Rows with t < 0 are skipped; a conv tap whose source row
// falls outside [0, L) contributes zeros (TF zero padding, reference modules.py:121-125).
// With R == L and jptr == nullptr this is the plain full-sequence case.
#pragma once
#include <vector>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>
#include <utility>

namespace dctts {

// Programmatic dependent launch (PDL): every kernel of the decode step starts with
// pdl_launch_dependents(); pdl_wait(); -- the next kernel's CTAs are scheduled while this one
// runs and only its main body waits for this grid's completion and memory flush.  That hides
// the kernel-to-kernel launch gap, which is what bounds the 50-kernel autoregressive step.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool& pdl_enabled();

template <typename... Params, typename... Args>
inline void launch_kernel(void (*kern)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
    if (e != cudaSuccess) throw std::runtime_error(std::string("kernel launch failed: ") + cudaGetErrorString(e));
}

struct RowWin {
    int B;            // batch
    int L;            // time length of the tensors
    int R;            // rows per batch element covered by this launch
    const int* jptr;  // device step index (window end), or nullptr -> L-1
};

struct ConvTap {
    const float* W;   // [K][ldw] row-major (output channel contiguous), zero padded to ldw
    int shift;        // source row = t + shift
};

// Y[orow][n] = bias[n] + sum_taps sum_k X[b, t+shift, k] * W_tap[k][n]
struct ConvArgs {
    const float* X; int ldx;
    float* Y; int ldy;             // pre-LN scratch, ldy == ldw (multiple of 4)
    const float* bias;             // [ldw], zero padded
    int K, N, ldw;
    int ntaps; ConvTap taps[3];
    RowWin win;
    int Lout, ostride, ooff;       // output row = b*Lout + t*ostride + ooff
    int accumulate = 0;            // tiled kernels only: Y += result (data gradient on top of the highway path)
};

// Dropout of the training step (modules.py:139 at training=True): a stateless hash of (dense element index, block index, seed) --
// TF's random stream cannot be reproduced, so the CPU checker and the kernels share this one (mix32).
struct DropArgs { uint32_t thresh = 0, layer = 0, seed = 0; float scale = 1.f; };   // keep iff mix32(i, layer, seed) >= thresh
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t mix32(uint32_t idx, uint32_t layer, uint32_t seed) {
    uint32_t x = idx * 0x9E3779B1u;
    x ^= layer * 0x85EBCA77u + seed;
    x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
    return x;
}
__device__ __forceinline__ float keep_mul(uint32_t idx, const DropArgs& d) {
    if (d.thresh == 0u) return 1.0f;
    return mix32(idx, d.layer, d.seed) >= d.thresh ? d.scale : 0.0f;
}
#endif

// Row-wise epilogue on the pre-LN scratch.
//  mode 0 (conv1d):  o = act(LN(y[0:C]) * g1 + b1);            out = o; out2 = sigmoid(o) if out2
//  mode 1 (hc):      H1 = sigmoid(LN(y[0:C])*g1+b1); H2 = LN(y[C:2C])*g2+b2;
//                    out = H1*H2 + (1-H1)*x
struct LnArgs {
    const float* Y; int ldy;       // scratch rows indexed like the output rows
    const float* g1; const float* b1; const float* g2; const float* b2;
    const float* X; int ldx;       // highway residual (mode 1), same row index as out
    float* out; int ldo;
    float* out2; int ldo2;         // optional sigmoid copy (mode 0)
    int C; int mode; int act;      // act: 0 none, 1 relu
    RowWin win;                    // rows are output rows: L here is the OUTPUT length
    int nparts = 1;                // split-K partials to sum (skinny GEMM), else 1
    int compact = 0;               // 1: scratch rows are indexed by b*R + r instead of the output row
    size_t part_stride = 0;        // floats between consecutive partials
    DropArgs drop;                 // training forward: dropout of the block output fused into this epilogue (thresh 0 = none)
};

struct GemmOut { int nparts; int compact; size_t part_stride; };

struct AttnArgs {
    const float* Q; int ldq;       // (B,T,d)
    const float* K; int ldk;       // (B,N,d)
    const float* V; int ldv;       // (B,N,d)
    float* Rout; int ldr;          // (B,T,2d) = [A.V ; Q]
    __half* r_hi; __half* r_lo; int ldr_h;   // optional split-plane copy of R for the tensor-core AudioDec
    float* align;                  // (B,N,T) or nullptr
    long long* maxatt;             // (B,T) or nullptr
    const int* pma;                // (B) window start, nullptr -> dense softmax over all keys
    int* p_next;                   // (B) or nullptr: argmax of row t_end
    int* p_hist;                   // (B,T) or nullptr: p_hist[b][t_end] = pma[b]
    int N, d, win_size;
    RowWin win;                    // rows = query rows (L = T)
};

// Griffin-Lim vocoder (kernels_vocoder.cu; reference utils.py:67-114)
struct VocoderArgs {
    const float* mag;          // (B, T, F) normalised linear magnitudes in [0, 1]
    float* S;                  // (B, T, F) amplitude target
    float2* X;                 // (B, T, F) complex spectrum estimate
    float* frames;             // (B, T, win) windowed time-domain frames
    float* wav;                // (B, hop*(T-1)) waveform (de-pre-emphasised at the end)
    float* mse;                // (B, 1 + Ly/512) frame energies for librosa.effects.trim
    const float2* tw; const float* window; const float* wss;
    double* deemph;                // (B, chunks) float64 states of the de-pre-emphasis recurrence
    int B, T, F, win, hop, n_iter;
    // ragged call: (B) DEVICE frame counts, 2 <= lengths[b] <= T; utterance b is computed as a call at T = lengths[b] alone
    // (its mag rows past it are not read, its samples past hop (lengths[b] - 1) are 0).  Null: every utterance has T.
    const int* lengths;
    const float* wsq;              // (n_fft) squared window centred in the frame: window sum-square past wss's valid range
    float max_db, ref_db, power;
    double preemphasis;            // float64 like the reference's scipy.signal.lfilter([1], [1, -hp.preemphasis], wav)
    // fast Griffin-Lim: E (B, T, F) the previous iteration's raw STFT estimate (zero before the first), updated in place;
    // alpha = momentum / (1 + momentum) rounded to float32.  Null E: the plain update.
    float2* E;
    float alpha;
    // spectral convergence: part (n_iter + 1, B, T) per-frame sums of (S - |est|)^2, conv (B, n_iter + 1) DEVICE float64.
    // Null part: no convergence, and no extra STFT of the final waveform.
    float* part;
    double* conv;
    // streaming step (dctts_vocoder_stream_push; null / 0 in every whole-signal call, which then launches the kernels'
    // STREAM = false instantiations, compiled to the code they had before these bounds existed).  lengths[b]
    // is the frames utterance b has received, and the launches cover only what the step changes, from (B) DEVICE bounds:
    //   prepare   mag (B, n_new, F) holds frames [new_lo[b], new_lo[b] + n_new); those below lengths[b] (not clamped) are set
    //   istft, stft_phase  frames [frame_lo[b], lengths[b]): n_active CTAs per utterance, frame frame_lo[b] + blockIdx.x
    //   ola       samples [sample_lo[b], hop (lengths[b] - 1)): n_samples per utterance; the samples below stay as they are
    //   deemph    samples [span[b].x, span[b].y) of deemph_in (B, Ly) into wav, from the float64 state state[b] (the output
    //             before span[b].x), which is replaced by the state at span[b].y - 1; n_span >= the longest span
    const int* new_lo;
    const int* frame_lo;
    const int* sample_lo;
    int n_new, n_active, n_samples;
    const int2* span;
    const float* deemph_in;
    double* state;
    int n_span;
};
// n_fft 1024, 2048 and 4096 have kernel instantiations (F = 1 + n_fft / 2 = 513, 1025, 2049); the launchers take n_fft
// from F and throw for any other size
bool voc_fft_size_ok(int n_fft);
// twiddles tw[k] = exp(-2 pi i k / n_fft) (n_fft entries), the win-tap Hann window, the window sum-square of T frames
// (n_fft + hop (T - 1) entries) and, when wsq_dev is given, the squared window it sums (n_fft entries)
void voc_make_tables(int n_fft, float2* tw_dev, float* window_dev, float* wss_dev, int T, int win, int hop, cudaStream_t s,
                     float* wsq_dev = nullptr);
// voc_run = voc_prepare, (voc_istft, voc_stft_phase) x n_iter, voc_istft, [voc_stft_phase, voc_convergence when part is
// set], voc_deemph, voc_energies
void voc_prepare(const VocoderArgs& a, cudaStream_t s);      // mag -> S, X = S (zero phase); 1 launch
void voc_istft(const VocoderArgs& a, cudaStream_t s);        // X -> frames -> wav; 2 launches
// wav, S (, E) -> X (, E); with part, iteration it's per-frame partials to part + it B T; 1 launch
void voc_stft_phase(const VocoderArgs& a, cudaStream_t s, int it = 0);
void voc_convergence(const VocoderArgs& a, cudaStream_t s);  // S, part -> conv; 1 launch
void voc_deemph(const VocoderArgs& a, cudaStream_t s);       // wav in place, deemph scratch; 3 launches
void voc_energies(const VocoderArgs& a, cudaStream_t s);     // wav -> mse; 1 launch
void voc_run(const VocoderArgs& a, cudaStream_t s);
int voc_launches_per_call(int n_iter, bool convergence = false);
size_t voc_deemph_scratch_bytes(int B, int T, int hop);
// feature extraction (reference utils.py:20-65,147-162) for a ragged batch of utterances packed back to back
struct FeatSeg {
    long long src;             // first sample of the utterance (after trimming, for feat_run) in the packed waveform
    int len;                   // its samples
    int f0;                    // its first frame in the flattened batch; entry B holds the total
};
struct FeatArgs {
    const void* wav; int dtype;        // packed waveform: 0 = float32, 1 = int16 PCM (value / 32768)
    const FeatSeg* seg; int B;         // DEVICE table of B + 1 entries
    int frames;                        // sum of the utterances' STFT frames (one CTA each)
    float* mag; float* mel;            // (B, mag_rows, F), (B, mel_rows, n_mels): frame t -> mag row t, mel row t / r if t % r == 0
    int mag_rows, mel_rows, r;
    const float* melw; const int* melrange; const float2* tw; const float* window;
    int F, n_mels, win, hop;
    float preemph, ref_db, max_db;
};
void feat_make_mel_basis(int sr, int n_fft, int n_mels, std::vector<float>& w, std::vector<int>& range);
void feat_frame_mse(const void* wav, int dtype, const FeatSeg* seg, int B, int frames, float* mse, cudaStream_t s);
void feat_run(const FeatArgs& a, cudaStream_t s);
// resampling in front of the features: librosa 0.6 core.resample(y, sr_orig, sr, res_type='kaiser_best', fix=True),
// i.e. resampy 0.2 resample / resample_f, for a ragged batch with one native rate per utterance
constexpr int RS_ZEROS = 64, RS_TABLE = 512, RS_NWIN = RS_ZEROS * RS_TABLE + 1;   // kaiser_best: 64 zeros, precision 9
struct ResampleUtt {
    long long src;             // first input sample in the packed waveform
    long long dst;             // first output sample in the packed output; entry B holds the total
    long long n_valid;         // int(n_in * ratio) samples resampy computes; [n_valid, next dst) are fix_length's zeros
    int n_in;                  // input samples
    int seg0, nseg;            // the utterance's time-register segments
    int index_step;            // int(scale * 512); 0: already at the output rate, only converted to float32
    double ratio, scale;       // sr_out / sr_in, min(1, ratio)
};
// The float64 time register of resample_f (time_register += time_increment once per output) for outputs
// [t0, next segment's t0): exactly v0 + (t - t0) * step.
struct TimeSeg {
    long long t0;
    double v0, step;
};
void resample_filter_table(std::vector<double>& win);
int resample_time_register(long long n_out, double inc, std::vector<TimeSeg>& out);
void resample_run(const void* wav, int dtype, const ResampleUtt* utt, int B, const TimeSeg* seg, const double* win, float* out,
                  long long total, cudaStream_t s);


// ---- training step (kernels_train.cu; reference train.py mode "train") ----
struct BlockBwdArgs {
    const float* pre; int ldy;         // pre-LN conv output (rows, nconv)
    const float* gout; int ldg;        // gradient w.r.t. the block output (rows, C), leading dimension ldg (also of gin)
    const float* X; int ldx;           // block input (highway residual), mode 1
    const float* g1; const float* b1; const float* g2; const float* b2;
    float* dy;                         // out: gradient w.r.t. the conv output (rows, nconv), leading dimension ldy
    float* gin;                        // out, mode 1: highway part of the input gradient (rows, C)
    float* dg1; float* db1; float* dg2; float* db2; float* dbias;   // accumulated (+=)
    long long rows; int C; int mode; int act;
    DropArgs drop;
};
struct WgradArgs {
    const float* X; int ldx; const float* dy; int ldy; float* dW; int ldw;
    long long rows; int L, K, N, ntaps; int shifts[3];
    int nsplit = 1, rows_per_split = 0;
};
struct AttnBwdArgs {
    const float* gR;                   // (B,T,2d) gradient of [ctx ; Q]
    const float* Q; int ldq; const float* K; const float* V; int ldkv;
    const float* align;                // (B,N,T) probabilities of the forward pass
    const float* gts; int ld_gts;      // guided-attention weights (max_N, max_T), row stride ld_gts; the (n_lim, t_lim) corner is read
    float* dS;                         // (B,T,N) scratch
    float* gQ;                         // (B,T,d)
    float* gKV;                        // (B,N,2d)
    int B, T, N, d; float att_scale;   // att_scale = 1 / (B n_lim t_lim)
    int n_lim, t_lim;                  // the guided-attention crop: min(N, max_N), min(T, max_T); keys / frames past it get no term
};
struct AdamEntry { float* p; float* g; float* m; float* v; long long n; };
// Ordered sums (option "train_deterministic", kernels_ordered.cu): a launcher given an OrderedWs writes every partial sum to
// `part` / `dpart` with plain stores in a fixed layout, then one ordered reduction adds the partials in a fixed order and
// does the single read-modify-write of the destination -- no float atomics, and no split count read from the device.
// Without one (nullptr) the launchers run the default kernels, which add with float atomics.  Every summing launcher
// returns the number of kernels it launched.
struct OrderedWs {
    float* part = nullptr; size_t part_elems = 0;      // weight-gradient and block-backward partials
    double* dpart = nullptr; size_t dpart_elems = 0;   // loss partials (ORD_LOSS_PARTS x 2)
};
constexpr int ORD_LOSS_CTAS = 1024;                    // fixed grid of the ordered loss kernels: at most this many partial rows
constexpr size_t ORD_LOSS_PARTS = 2 * ORD_LOSS_CTAS;   // doubles of OrderedWs::dpart
// floats of OrderedWs::part the ordered path of each launcher needs (0: it adds each element once and needs none)
size_t block_bwd_ordered_floats(long long rows, int C, int mode);
size_t conv_wgrad_ordered_floats(const WgradArgs& w);
size_t conv_wgrad_tc_ordered_floats(const WgradArgs& w, int B);
int conv_wgrad_ordered_splits(const WgradArgs& w);    // row splits of the fp32 weight gradient in the ordered mode
void launch_train_dropout(float* x, long long rows, int C, int ld, const DropArgs& d, cudaStream_t s);
int launch_train_loss(const float* logits, int ldl, const float* target, float* dlogits, int ldg, double* sums, long long rows, int C,
                      cudaStream_t s, const OrderedWs* ord = nullptr);
int launch_train_block_bwd(const BlockBwdArgs& a, cudaStream_t s, const OrderedWs* ord = nullptr);
int launch_conv_wgrad(WgradArgs a, cudaStream_t s, const OrderedWs* ord = nullptr);
void launch_transpose_w(const float* W, float* WT, int ntaps, int K, int N, int ldw, int Kp, cudaStream_t s);
int launch_attn_bwd(const AttnBwdArgs& a, double* sums, cudaStream_t s, const OrderedWs* ord = nullptr);
// what launch_attn_bwd refuses before it launches anything: d != 256, a crop outside (N, T) or wider than the table's stride
void check_attn_bwd(const AttnBwdArgs& a);
// the guided-attention sum alone (the first kernel(s) of launch_attn_bwd): sums[2] += sum over the (n_lim, t_lim) corner of |A gts|
int launch_attn_loss(const float* align, const float* gts, int ld_gts, double* sums, int B, int N, int T, int n_lim, int t_lim,
                     cudaStream_t s, const OrderedWs* ord = nullptr);
// out (rows, C) dense = sigmoid(x), x (rows, C) with leading dimension ldx
void launch_sigmoid_rows(const float* x, int ldx, float* out, long long rows, int C, cudaStream_t s);
void launch_guided_attention(float* W, int N, int T, cudaStream_t s);
// dtable[id] += g[row] for every row with ids[row] = id in [1, vocab) (row 0 of the table gets no gradient)
int launch_embed_bwd(const int* ids, const float* g, float* dtable, int rows, int e, int vocab, cudaStream_t s,
                     const OrderedWs* ord = nullptr);
void launch_adam(const AdamEntry* entries_dev, int n_entries, float lr_t, float beta1, float beta2, float eps, cudaStream_t s);
// the ordered kernels behind the launchers above (kernels_ordered.cu)
template <int MAXV, bool HC> int launch_train_block_bwd_ordered(const BlockBwdArgs& a, const OrderedWs& o, cudaStream_t s);
int launch_conv_wgrad_ordered(const WgradArgs& a, const OrderedWs& o, cudaStream_t s);     // a.nsplit, a.rows_per_split set
int launch_train_loss_ordered(const float* logits, int ldl, const float* target, float* dlogits, int ldg, double* sums, long long rows,
                              int C, const OrderedWs& o, cudaStream_t s);
int launch_attn_loss_ordered(const float* align, const float* gts, int ld_gts, double* sums, int B, int N, int T, int n_lim, int t_lim,
                             const OrderedWs& o, cudaStream_t s);
int launch_embed_bwd_ordered(const int* ids, const float* g, float* dtable, int rows, int e, int vocab, cudaStream_t s);
// dst += the sum over p of part[p][0, width), split into up to 5 destinations: column col0 + i of a segment goes to
// dst[(i / n) ld + i % n] when i % n < w (partial rows padded past a destination row's w columns skip the padding)
struct ColSeg { void* dst = nullptr; long long col0 = 0; int n = 1, w = 1, ld = 1; };
struct ColSegs { int nseg = 0; ColSeg s[5]; };
template <typename T> void launch_ordered_colsum(const T* part, long long nparts, long long width, const ColSegs& sg, cudaStream_t s);

// ---- the training GEMMs on wgmma (kernels_gemm_tc.cu): drop-ins for launch_conv_gemm (tiled path) / launch_conv_wgrad ----
struct GemmTcWs {
    __half* a_hi = nullptr; __half* a_lo = nullptr; size_t a_elems = 0;   // operand A planes (activations / gradients, plain or transposed)
    __half* b_hi = nullptr; __half* b_lo = nullptr; size_t b_elems = 0;   // operand B planes (weights / transposed gradients)
    unsigned* slots = nullptr; int n_slots = 0; int cursor = 0;           // per-tensor abs-max slots, cleared once per step
    int probe = 0;                                                        // measurement only: fetch the operands, issue no MMA, store nothing
};
void gemm_tc_begin_step(GemmTcWs& ws, cudaStream_t s);
bool conv_gemm_tc_ok(const ConvArgs& c, const GemmTcWs& ws);
struct GemmTcSlots { unsigned* x = nullptr; unsigned* w = nullptr; };   // in: abs-max already known (same tensor converted earlier this step); out: the slots used
int launch_conv_gemm_tc(const ConvArgs& c, GemmTcWs& ws, cudaStream_t s, GemmTcSlots* io = nullptr);
bool conv_wgrad_tc_ok(const WgradArgs& w, int B, const GemmTcWs& ws);
int launch_conv_wgrad_tc(const WgradArgs& w, int B, GemmTcWs& ws, cudaStream_t s, GemmTcSlots* io = nullptr, const OrderedWs* ord = nullptr);

// ---- weight packers (kernels_pack.cu): fp32 W [tap][cin][ldw] -> wgmma planes and the persistent decode's stream ----
constexpr int PACK_MAXL = 64;  // layers of one abs-max launch (the four networks have 54)
struct PackMaxTable { const float* W[PACK_MAXL]; long long n[PACK_MAXL]; int count; };
// maxbits_dev[e] = float bits of max |W| over the n[e] floats at W[e]; the caller zeroes maxbits_dev first
void launch_weight_absmax(const PackMaxTable& t, unsigned* maxbits_dev, cudaStream_t s);
struct TcPackArgs {           // LayerDev::TcPack's geometry; hi / lo: [nrows][Ktot]; W pre-multiplied by scale
    const float* W; __half* hi; __half* lo;
    int mode, cin, cout, ldw, cin_pad, Ktot, nrows, bn, half; float scale;
};
void launch_pack_tc(const TcPackArgs& a, cudaStream_t s);
struct DecPackArgs {          // one decode block: K = ntaps * cinp k rows in chunks of krows at rank float offsets off (fp32) / off16 (slabs)
    const float* W; float* stream; int stream_len;
    int kind, cin, cout, ldw, cinp, K, krows, ns, cs, off, off16;
    float scale;              // > 0: also the split-fp16 MMA slabs of a receptive-field block, W pre-multiplied by scale
};
void launch_pack_decode(const DecPackArgs& a, cudaStream_t s);

// scratch_bytes bounds the split-K partial buffer of the skinny path
GemmOut launch_conv_gemm(const ConvArgs& a, cudaStream_t s, size_t scratch_bytes, bool allow_skinny = true);
void launch_ln_rows(const LnArgs& a, cudaStream_t s);
bool conv_gemm_ln_fusable(const ConvArgs& a, const LnArgs& n);
void launch_conv_gemm_ln(const ConvArgs& a, LnArgs n, int* tickets, cudaStream_t s, size_t scratch_bytes);
void launch_attention(const AttnArgs& a, cudaStream_t s);
void launch_embed(const int* ids, const float* table, float* out, int rows, int e, cudaStream_t s);
// p_cur = p_next; j += 1  (end of an AR step)
void launch_ar_advance(int* p_cur, const int* p_next, int* j, int B, cudaStream_t s);
void launch_ar_advance_path(int* p_cur, const int* p_next, int* j, const int* path, int* amax_hist, int B, int T, cudaStream_t s);
void launch_fill_i32(int* p, int v, int n, cudaStream_t s);

// ---- the aligner's monotonic path search (kernels_align.cu; DESIGN.md section 4d) ----
struct AlignArgs {
    const float* A;                // (B, N, T) alignments
    const int* meta;               // (2B): the frames T_b of every utterance, then its text end e_b
    unsigned char* bp;             // (B, T, N) back-pointer workspace
    int* path; int* chars;         // (B, T) out, -1 past T_b
    int* durations;                // (B, N) out
    double* score;                 // (B) out: D[e_b, T_b - 1]
    int B, N, T, win;
};
// one CTA per utterance with 2 (max_end + 1) doubles of dynamic shared memory; 1 launch
void launch_align_search(const AlignArgs& a, int max_end, cudaStream_t s);

// ---- mel-cepstral distortion along a DTW alignment (kernels_mcd.cu; DESIGN.md section 8h) ----
struct McdArgs {
    const float* X; const float* Y;    // (B, Tx, n_mels), (B, Ty, n_mels) dB-normalised mels
    const long long* meta;             // (4B): nx_b, ny_b, back-pointer offset, cepstrum workspace offset (-1: shared memory)
    const double* dct;                 // (K, n_mels): rows 1 .. K of the orthonormal DCT-II matrix
    double* cep;                       // cepstra of the pairs that do not fit in shared memory, rows of K | 1 doubles
    unsigned char* bp;                 // back-pointers, nx_b ny_b bytes per pair
    double* mcd; int* pairs;           // (B) out
    int* path;                         // (B, Tx + Ty - 1, 2) out (i, j), -1 past pairs[b]; may be null
    double max_db, ref_db;
    int B, Tx, Ty, n_mels, K;
};
// one CTA per pair with `smem` bytes of dynamic shared memory; 1 launch
void launch_mcd_dtw(const McdArgs& a, size_t smem, cudaStream_t s);

// ---- the long-form join of decoded pieces into one mel sequence per text (kernels_longform.cu; DESIGN.md section 4e) ----
struct JoinArgs {
    const float* Y;                    // (P, T, C) the decoded pieces
    const int* len;                    // (P) rows of each piece (clamped to [0, T])
    const int* text;                   // (P) the text of each piece; a text's pieces are consecutive and in order
    const int* pause;                  // (P) rows of `silence` after each piece, 0 after a text's last piece
    const int* first;                  // (K + 1) the first piece of each text, then P
    float* out;                        // (K, T_out, C)
    int* out_len;                      // (K) rows of each text's sequence
    float silence;
    int P, K, T, C, T_out;
};
// one CTA per piece; 1 launch
void launch_join_rows(const JoinArgs& a, cudaStream_t s);

}  // namespace dctts
