// kernels_tc.cuh -- interface of the wgmma fused conv + LayerNorm / highway kernels.
//
// Activations on the tensor-core path are split-fp16 planes (numerics.cuh).  The audio-level input of AudioEnc, AudioDec
// and SSRN is scaled per utterance (launch_f32_to_planes_scaled), undone in the first block's epilogue.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace dctts {

struct Planes {
    __half* hi = nullptr;
    __half* lo = nullptr;
    int ld = 0;           // elements per row (multiple of 8 -> 16-byte rows for TMA)
};

struct TcArgs {
    // epilogue parameters
    const float* bias;             // [nconv] original (TF) column order
    const float* g1; const float* b1; const float* g2; const float* b2;
    int mode;                      // 0 conv1d (one LN), 1 hc (two LNs + gate + mix), 2 transposed conv (two LNs, two rows)
    int act;                       // mode 0: 0 none, 1 relu
    int C;                         // LN width (mode 0: cout; modes 1,2: cout of one half)
    int bn;                        // accumulator columns per CTA (modes 1,2: both halves): 64, 80, 144 or 256
    int half;                      // columns per LN half per CTA (mode 0: == bn)
    float inv_scale;               // 1 / (power-of-two weight scale)
    const float* in_inv;           // [B] 1 / (power-of-two scale of utterance b's input planes), or null for unscaled
                                   // planes; modes 0 and 2 only (hc reads its residual from the input planes as is)
    // reduction schedule
    int ntaps; int shifts[3]; int kb_per_tap; int stages;   // kb_per_tap in units of the kernel's BK (64 or 32)
    int mcast;                     // 1: the A tile is fetched once per cluster (each CTA loads 128/ncta rows, TMA multicast)
    int resid_tma;                 // 1 (hc): residual tile via TMA into its own shared-memory tile
    int out_tma;                   // 1 (hc, full sequences, needs resid_tma): output planes staged in that stage and TMA-stored
    // tiling: 128 rows = TT time rows x TB batch rows
    int TT, TB, tiles_t, ntiles;   // ntiles = batch groups x tiles_t (one tile per CTA row of the grid)
    RowWin win;
    // residual (mode 1) and outputs
    Planes X;                      // highway residual, same row index as the output
    Planes out;                    // split-plane output (may be null)
    float* out_f32; int ld_f32;    // fp32 output (may be null)
    float* sig_f32; int ld_sig;    // fp32 sigmoid(output) (mode 0, may be null)
    Planes sig;                    // split planes of sigmoid(output) (mode 0, may be null)
    // per-utterance lengths (ragged SSRN): utterance b's rows t >= lengths[b] << len_shift (input rows; mode 2 writes both
    // output rows 2t and 2t+1) are stored as zeros.  Null: every row of the launch is live.
    const int* lengths; int len_shift;
    int* dbg;                     // optional host-mapped progress markers (debugging), else null
};

// Encodes the rank-3 (C, L, B) activation map with a {bk, TT, TB} box; bk = 64 -> 128-byte swizzle, 32 -> 64-byte.
void tc_make_act_map(CUtensorMap* m, const __half* base, int C, int ld, int L, int B, int TT, int TB, int bk);
// Encodes the rank-2 (Ktot, Nrows) K-major weight map with a {bk, bn} box, same swizzle rule.
void tc_make_w_map(CUtensorMap* m, const __half* base, int Ktot, int Nrows, int bn, int bk);

// Generic rank-3 fp16 map {d0 (contiguous), d1, d2} with byte strides and a {b0, b1, 1} box (b0 = 32 or 64 halfs).
void tc_make_map3(CUtensorMap* m, const __half* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                  uint64_t stride2_bytes, uint32_t b0, uint32_t b1);

// pipeline depth that fits the shared-memory budget for `bn` accumulator columns per CTA (with or without the residual tile)
int tc_stages_for(int bn, int bk, int resid_tma, int half);
// reduction slab per pipeline stage (fp16 elements): 32 (64B swizzle)
int tc_bk();
// co-resident clusters of `ncta` CTAs of the conv1d instantiation with `bn` columns (0: none can be scheduled)
int conv_ln_tc_max_clusters(int ncta, int bn, int bk);
// grid = (ncta, tiles); cluster (ncta,1,1)
void launch_conv_ln_tc(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi,
                       const CUtensorMap& w_lo, const CUtensorMap* io /* [4]: X hi, X lo, out hi, out lo ({64,128,1} boxes) or null */, const TcArgs& a, int ncta, int ctas_y, int bk, cudaStream_t s);

// ---- wgmma attention (kernels_attn_tc.cu) ----
struct AttnTcArgs {
    const float* Q; int ldq;       // fp32 queries (copied verbatim into R[:, d:2d])
    float* R; int ldr;             // (B,T,2d) = [A.V ; Q]
    Planes Rpl;                    // optional split-plane copy of R
    float* align;                  // (B,N,T) or nullptr
    long long* maxatt;             // (B,T) or nullptr
    const int* pma;                // (B) monotonic window start, nullptr -> dense softmax
    int T, N, d, win_size;
    float scale;                   // 1/sqrt(d)
};
// keys of the transposed V planes: N rounded up to the kernel's 64-key block
int attn_tc_padded_keys(int N);
// K, V fp32 -> K planes (B,N,d) and transposed V planes (B,d,vtp.ld), vtp.ld >= attn_tc_padded_keys(N), keys >= N zero
void launch_attn_kv_planes(const float* K, int ldk, const float* V, int ldv, Planes kp, Planes vtp, int B, int N, int d,
                           cudaStream_t s);
void launch_attention_tc(const Planes& Q, const Planes& K, const Planes& Vt, const AttnTcArgs& a, int B, cudaStream_t s);

void launch_f32_to_planes(const float* x, int ldx, Planes p, long long rows, int C, cudaStream_t s);
// (B, L, C) fp32 -> planes of s_b x with s_b = utterance_scale(max |x_b|) (numerics.cuh); in_inv[b] = 1 / s_b for
// TcArgs::in_inv.  No host sync.  lengths (device, optional): only utterance b's rows t < lengths[b] are read (the scale is
// their abs-max), its rows past them become zero planes.
void launch_f32_to_planes_scaled(const float* x, int ldx, Planes p, int B, int L, int C, float* in_inv, cudaStream_t s,
                                 const int* lengths = nullptr);
void launch_planes_to_f32(Planes p, float* y, int ldy, long long rows, int C, cudaStream_t s);
// Windows of mel rows for the windowed SSRN of a synthesis stream: window w is rows [row0[w], row0[w] + len[w]) of
// utterance utt[w] of Y (B, T, C) fp32, as rows [0, len[w]) of a (W, L, C) plane batch at the fixed scale
// SSRN_WINDOW_SCALE; rows [len[w], L) become zero planes.  in_inv[w] = 1 / SSRN_WINDOW_SCALE.  win: len[W] | utt[W] | row0[W]
// (device ints).  The scale is utterance_scale's for an abs-max in [0.5, 1), which a sigmoid output below 1 reaches
// whenever its loudest value is >= 0.5: then the planes equal launch_f32_to_planes_scaled's on the whole utterance.
constexpr float SSRN_WINDOW_SCALE = 32768.f;
void launch_mel_windows_to_planes(const float* Y, int T, int C, const int* win, int W, int L, Planes p, float* in_inv,
                                  cudaStream_t s);

}  // namespace dctts
