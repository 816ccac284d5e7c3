// kernels_decode.cuh -- the autoregressive Text2Mel decode loop (reference synthesize.py:45-54) as ONE
// persistent launch: a 16-CTA thread-block cluster per group of <= 5 utterances walks AudioEnc ->
// Attention -> AudioDec for all mel frames, streaming its slice of the 27 MB of decode weights
// from L2 through a TMA-bulk ring.  See kernels_decode.cu for the design.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dctts {

constexpr int DEC_NC = 16;          // CTAs per cluster (non-portable cluster size)
constexpr int DEC_GMAX = 5;         // utterances per cluster (the benchmark's 32 utterances need 7 co-resident 16-CTA clusters)
constexpr int DEC_THREADS = 256;
constexpr int DEC_NSLOT = 3;        // ring slots
constexpr int DEC_REG_F = 1536;     // floats per warp region of a slot (6 KB): every warp streams and frees its own k-rows
constexpr int DEC_SLOT_F = 8 * DEC_REG_F;   // 48 KB per slot
constexpr int DEC_MAXL = 24;        // 13 AudioEnc + 11 AudioDec blocks
constexpr int DEC_MAXCH = 48;       // weight chunks per frame
constexpr int DEC_PRM_F = 1024 + 64;   // per-layer parameter block: gamma1 | beta1 | gamma2 | beta2 (256 each) | bias slice
constexpr int DEC_PL_PAD = 88;      // zero rows in front of t = 0 in the split-fp16 plane histories (>= the tallest source window: 84 rows)
constexpr int DEC_NPROF = 24;       // lap-timer buckets (option decode_prof; dctts_decode_profile lists them)

struct DecLayer {
    int kind;        // 0 conv1d (LN, optional relu), 1 hc (two LNs, sigmoid gate, highway mix)
    int cin;         // input channels
    int cout;        // output channels (256, or n_mels for the last block)
    int ntaps, rate; // causal taps at t - (ntaps-1-i)*rate
    int act;         // 1 = relu (conv1d)
    int ns;          // weight-slice columns per CTA (multiple of 4)
    int cs;          // channels owned per CTA (per LN half)
    int ch0, nch;    // chunk range of this layer within a frame
    int krows;       // k rows per chunk of this layer
    int prow;        // AudioDec receptive-field rows to recompute when the attention window moved (1 otherwise)
    int ldin;        // leading dimension of the input history
};
struct DecChunk { int off; int off16; short nfl4; short k0; short krows; short layer; };   // off: float offset in a rank's stream (off16: of the
                                                                   // same rows as split-fp16 MMA slabs); nfl4: floats / 4; k0: first k row (tap*cin + ci)

struct DecParams {
    DecLayer L[DEC_MAXL];
    DecChunk C[DEC_MAXCH];
    const float* in_hist[DEC_MAXL];    // (B, T, cin) history of the layer's input (nullptr: lives in shared memory only)
    float* out_hist[DEC_MAXL];         // (B, T, cout) history of the layer's output
    const float* lnp[DEC_MAXL];        // [4][256] gamma1, beta1, gamma2, beta2
    const float* bias[DEC_MAXL];       // [nconv] in the TF column order (gate | info for hc)
    const float* wstream;              // [DEC_NC][stream_len] packed weight slices, chunk by chunk
    const float* kv;                   // (B, N, 2d): K | V
    float* ybuf;                       // (B, T, n_mels)
    float* rbuf;                       // (B, T, 2d)
    float* pre_scr;                    // [clusters][G * max prow][512] pre-LN scratch of the recompute path
    // The recompute path's A operand: the layer's input history a second time as split-fp16 planes in the wgmma no-swizzle
    // K-major slab layout, per utterance [cin/16 slabs][plane hi, lo][k8 group][DEC_PL_PAD + T rows][8 halfs]; the first
    // DEC_PL_PAD rows stay zero (TF's causal zero padding).  nullptr for layers the recompute does not read this way.
    __half* pl_hist[DEC_MAXL];
    __half* pl_c1;                     // [clusters * G][cin/16][2][2][DEC_PL_PAD][8]: the recomputed rows of the first AudioDec block's input
    int pl_rows;                       // DEC_PL_PAD + T
    int* p_hist;                       // (B, T) window used at every step
    int* p_final;                      // (B) window after the last step
    float inv_scale[DEC_MAXL];         // 1 / (power-of-two scale of the block's split-fp16 weight planes), tensor-core pre-pass
    int* stats;                        // [clusters][2]: frames with a window move, utterance-frames recomputed
    long long* prof;                   // optional [DEC_NPROF] SM-clock lap timers of cluster 0 / rank 0 (option decode_prof), else nullptr
    int nl, n_enc, nch, nch_enc, pyr_ch0, pyr_ch1, stream_len;   // pyr_ch0..pyr_ch1: chunks of the AudioDec blocks with prow > 1
    int B, G, T, N, d, n_mels, win_size, steps;
    int force_prepass;                 // option decode_force_prepass: every utterance recomputes at every frame j >= 1
    // End of utterance (decode_until_kernel only; nullptr / unused in decode_cluster_kernel): utterance b ends `tail` frames
    // after the first frame whose attention argmax reaches stop_pos[b] (< 0: never); a cluster leaves the frame loop once
    // all its utterances have ended.
    const int* stop_pos;               // (B)
    int* lengths;                      // (B) out: frames of each utterance
    int* frames;                       // [clusters] out: frames the cluster executed
    int tail;
};
static_assert(sizeof(DecParams) <= 4000, "DecParams must fit the kernel parameter space");

size_t decode_smem_bytes();
// returns cudaSuccess or the launch / attribute error (the caller decides whether to fall back).
// p.stop_pos != nullptr runs decode_until_kernel (end of utterance, no lap timers).
cudaError_t launch_decode_cluster(const DecParams& p, int n_clusters, cudaStream_t s);
// decode_path_kernel: frame j of utterance b runs under the window path[b * T + j] (frame 0 included) instead of the
// previous frame's argmax, which goes to amax_hist[b * T + j].  p.lengths (B) are inputs, 1 <= lengths[b] <= p.steps, and
// a cluster executes the longest of its utterances (p.frames as decode_until_kernel; p.stop_pos is not read).
cudaError_t launch_decode_path(const DecParams& p, const int* path, int* amax_hist, int n_clusters, cudaStream_t s);
// decode_progress_kernel: decode_until_kernel (p.stop_pos, p.lengths, p.frames required) that, at the end of every frame,
// publishes to progress[c * DEC_PROG_INTS + ...] (host memory mapped into the device) cluster c's frames done (int 0,
// release store at system scope) and each of its utterance slots' length, -1 while unknown (ints 1 .. DEC_GMAX).  Y rows
// of frames below the count are visible to a host thread that read the count with acquire.
constexpr int DEC_PROG_INTS = 8;
cudaError_t launch_decode_progress(const DecParams& p, int* progress, int n_clusters, cudaStream_t s);
// Rows past each utterance's length: Y (B, T, n_mels) rows 0, prev_hist (B, T) rows -1 (either may be nullptr).  With
// `derive`, lengths[b] is first computed from the window history p_hist (B, T) of a run of `steps` frames by the rule
// decode_until_kernel applies in its frame loop.
void launch_until_finish(const int* stop_pos, int tail, int steps, int T, int n_mels, const int* p_hist, bool derive,
                         int* lengths, float* Y, int* prev_hist, int B, cudaStream_t s);
// 0 when a 16-CTA cluster with this shared-memory footprint cannot be scheduled on the current device
int decode_max_active_clusters();

}  // namespace dctts
