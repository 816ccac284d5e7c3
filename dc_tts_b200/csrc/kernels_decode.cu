// kernels_decode.cu -- the whole autoregressive decode (reference synthesize.py:45-54: 210 x
// {AudioEnc, Attention, AudioDec}, networks.py:73-212) in ONE persistent launch.
//
// Why: a decode step is 24 dependent conv blocks on one row per utterance; as 46 graph nodes it was
// bound by kernel boundaries and by split-K round trips through L2 (round 1: ~300 us per step, 1.5 %
// of any roofline).  Utterances never interact (networks.py:140-153 is batched per row), so a group
// of G <= 5 utterances is decoded by one thread-block CLUSTER with no grid-level synchronisation:
//
//   * 16 CTAs per cluster; CTA r owns 1/16 of every block's output channels (for `hc` the same 16
//     channels of the gate and of the info half, so the highway mix is local).
//   * its weight slices for all 24 blocks form one contiguous 1.7 MB stream (packed at commit time).
//     The stream is the same for every frame and is pulled from L2 by TMA bulk copies
//     (cp.async.bulk + mbarrier) into a 3 x 48 KB shared-memory ring.  Every WARP owns the k rows it
//     multiplies: it waits on its own mbarrier, and refills its own 6 KB region the moment it has read
//     it -- the chunk loop has no block-wide synchronisation at all.
//   * per block: GEMV of the slice on fp32 FMA (exact fp32 arithmetic, as the reference), one block
//     barrier for the cross-warp reduction; the threads that finish the slice's values store them from
//     registers into every peer with st.async through distributed shared memory, together with the
//     LayerNorm statistics of the slice's channels, completing on the peer's mbarrier (no hardware
//     cluster barrier on this path); every CTA then merges the 16 slices' statistics and normalises the
//     whole rows redundantly (gate / highway mix one thread per channel), so the next block's input is
//     in local shared memory.  Two block barriers per block.  Dilated taps come from the per-layer
//     history in HBM/L2, prefetched one block ahead with cp.async while the peers' slices are in
//     flight; each CTA appends its channel slice of the new row.
//   * Quirk Q1 (SURVEY 3.1): the reference recomputes R under the CURRENT window every step.  While
//     the window of an utterance does not move, the cached rows are exactly what a recompute would
//     give.  When it moves, a PRE-PASS refreshes the rows t < j of its AudioDec receptive field
//     (84/82/76/58/4/2 rows of C_1, HC_2..HC_6) under the new window -- attention one warp per row, a
//     wgmma GEMM per utterance (split-fp16 planes staged per 16-channel slab in the no-swizzle K-major
//     layout, each slab fetched once per cluster and multicast to its 16 CTAs, the three taps being the
//     same slab read through shifted descriptors), pre-LN rows through
//     an L2 scratch, LayerNorm one warp per row over the whole cluster -- and the ordinary one-row pass
//     then runs for every utterance.  The pre-pass consumes the same weight chunks a second time: the
//     stream is "virtual" (frame, segment, chunk) and both the consumer and the refill cursor walk it.
//
// All waits are bounded (mbarrier waits trap after ~2 s).  Hardware cluster barriers (pre-pass, frame
// end) are executed by all threads of all CTAs in uniform control flow: every branch that contains
// one depends only on the attention windows, which every CTA computes identically.
#include "kernels_decode.cuh"
#include "numerics.cuh"
#include "tc_ptx.cuh"

#include <cuda_fp16.h>
#include <atomic>
#include <cstddef>
#include <math.h>

namespace dctts {
using namespace ptx;

namespace {

constexpr int NC = DEC_NC, GMAX = DEC_GMAX, NT = DEC_THREADS, NWARP = NT / 32;
constexpr int XLD = 768;                       // row pitch of the input vectors: [tap0 | tap1 | current]
constexpr int PLD = GMAX * 32 + 16;            // pitch between the ranks' slices in `pre` (16 floats of bank skew)
constexpr int PPD = 2 * NC + 4;                // pitch of one (utterance, LN half) in `part`: NC x (mean, M2), 4 floats of bank skew
constexpr int TC_RA = DEC_PL_PAD;              // pre-pass: rows per k8 group of an A slab plane (source rows per utterance, decode_tables)
constexpr int TC_APLANE = 2 * TC_RA * 16;      // bytes of one plane of one 16-channel slab (2 k8 groups)
constexpr int TC_ASTAGE = 2 * TC_APLANE;       // hi + lo planes
constexpr int TC_NSTG = 6;                     // A slab stages: five slabs in flight while one is multiplied
constexpr int gcd_c(int a, int b) { return b == 0 ? a : gcd_c(b, a % b); }
constexpr unsigned TC_QCYC = NC / gcd_c(NC, TC_NSTG) * TC_NSTG;   // slabs between two stagings of one stage by one CTA
constexpr int TC_PR = 24;                      // packed tile (pyr_tc_packed): rows per k8 group of a tap image (>= GMAX * 4)
constexpr int TC_PTAP = 2 * 2 * TC_PR * 16;    // bytes of one tap image (hi + lo planes, 2 k8 groups)
static_assert(3 * TC_PTAP <= TC_ASTAGE, "packed tap images inside a stage");
static_assert(GMAX * NT >= 1024, "red: LayerNorm parameters of the pre-pass");
static_assert(TC_RA == DEC_PL_PAD, "pl_c1 rows are staged as whole slabs");

struct Smem {
    float ring[DEC_NSLOT][NWARP][DEC_REG_F];
    float red[GMAX][NT];                // per-frame path: partial sums per warp; pre-pass: LayerNorm parameters of the block
    float xin[2][GMAX][XLD];
    union {                             // never live together: between the cluster barriers that enclose the pre-pass no peer
                                        // sends pre-LN slices, so the pre-pass stages A here (and the peers' multicast
                                        // slabs land here only between those barriers)
        struct {
            float pre[2][NC][PLD];
            float part[2][GMAX * 2][PPD];   // every rank's LayerNorm partials (mean, M2) per (utterance, LN half)
        };
        unsigned char tca[TC_NSTG][TC_ASTAGE];   // (the MMAs read up to 128 + 54 rows past a slab start: prm follows)
    };
    float prm[2][DEC_PRM_F];
    unsigned long long fullw[DEC_NSLOT][NWARP];
    unsigned long long gbar[2];
    unsigned long long sbar[TC_NSTG], abar[TC_NSTG];   // pre-pass: slab stage free / slab stage filled
    uint32_t tc_baddr[96];              // pre-pass: descriptor start field of every weight slab of the current block
    int n_moved_frames, n_moved_utt;
    DecParams P;                        // the kernel's parameter block: indexed per block / chunk on the critical path; in the
                                        // constant bank those indexed loads missed the (instruction-shared) constant cache
    int p_cur[GMAX], p_prev[GMAX], p_next[GMAX], moved[GMAX];
    int fmoved[2];
    long long prof[DEC_NPROF], prof_last;
    int stop[GMAX], ulen[GMAX], f_end;  // decode_until_kernel: stop positions, lengths (-1 while unknown), frames to execute
};

static_assert(sizeof(Smem) + 128 <= 232448, "decode kernel: shared memory budget (227 KB per CTA)");
// An A descriptor reads 64 rows per live M half from its k8 group: up to TC_RA + 128 rows from a group that holds TC_RA
// (tap shift <= TC_RA, decode_tables), i.e. up to 128 rows of 16 bytes past the end of the last stage.  Those rows are thrown
// away but must be shared memory of this kernel.
static_assert(offsetof(Smem, tca) + sizeof(Smem::tca) + 128 * 16 <= sizeof(Smem), "A tile reads past the stages");
static_assert(offsetof(Smem, pre) % 16 == 0 && (PLD * 4) % 16 == 0, "pre: 16-byte st.async targets");
static_assert(offsetof(Smem, part) % 16 == 0 && (PPD * 4) % 16 == 0, "part: float4 loads of the merge");

// lap timer (option decode_prof): thread 0 attributes the cycles since the previous lap to bucket i
#define LAP(i) do { if constexpr (PROF) { if (threadIdx.x == 0) { const long long now_ = clock64(); S.prof[i] += now_ - S.prof_last; S.prof_last = now_; } } } while (0)
enum { LP_START = 0, LP_WAIT = 1, LP_GEMV = 2, LP_RELEASE = 3, LP_GATHER = 4, LP_CBAR = 5, LP_LN = 6, LP_MIX = 7, LP_ATT = 8,
       LP_PYR_ATT = 9, LP_PYR_WTS = 10, LP_PYR_TABLE = 11, LP_PYR_STAGE = 12, LP_PYR_DRAIN = 13, LP_PYR_REFILL = 14,
       LP_PYR_LN = 15, LP_PYR_BAR = 16, LP_FRAME = 17,
       // the MMA warpgroup's own laps (thread 128, pyr_mma_rows): they overlap thread 0's
       LP_WG_AWAIT = 18, LP_WG_MMA = 19, LP_WG_EPI = 20,
       // thread 0 again: issuing the next block's parameter and tap prefetch, between its slice stores and the gather wait
       LP_PREFETCH = 21, LP_COUNT };
static_assert(LP_COUNT <= DEC_NPROF, "lap buckets");

// NOTE on `__noinline__` in this file: there is none.  With 227 KB of shared memory per CTA the L1 data cache is ~0 KB, so every
// stack access (ABI spills of a non-inlined call, a dynamically indexed local array) is an L2 round trip of ~500 cycles: the
// first three versions of this kernel spent 60 % of their time there (ptxas must report a 0-byte stack frame).
// the per-frame path: ex2.approx + rcp (2 ulp each; far inside the 1e-3 budget, half the instructions)
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;                                   // 0: zero fill (TF zero padding of the causal conv)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// the same, multicast: the bytes land at the same CTA-relative offset in every CTA of `mask`, each completing on its own
// mbarrier at the offset of `bar`
__device__ __forceinline__ void bulk_g2s_mc(void* dst, const void* src, uint32_t bytes, unsigned long long* bar, uint16_t mask) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() { cluster_arrive(); cluster_wait(); }

// The progress of one cluster after frame j (decode_progress_kernel; rank 0, thread 0, after the frame's closing
// cluster_sync_all): p[1 + g] = S.ulen[g] (-1 while utterance g's length is unknown), then p[0] = j + 1 frames done.
// p is host memory mapped into the device; the host reads p[0] with acquire and then p[1..].
// Memory ordering: Y is written only by rank 0 (layer_row's last block, one thread per channel), and every thread of
// rank 0 -- every thread of the cluster -- has passed barrier.cluster.arrive.release of this frame's closing barrier before
// this thread's wait.acquire returned.  So this frame's Y rows, and the other 15 CTAs' history rows (which the host never
// reads), happen before the fence in causality order; fence.sc.sys then orders them, and the lengths below, before the
// release store of the count at system scope.  A host thread that reads the count with acquire and then launches work
// that reads ybuf sees every Y row of frames < count.
__device__ __forceinline__ void publish_progress(int* p, int frames, const int* ulen) {
#pragma unroll
    for (int g = 0; g < DEC_GMAX; ++g) asm volatile("st.relaxed.sys.u32 [%0], %1;" :: "l"(p + 1 + g), "r"(ulen[g]) : "memory");
    __threadfence_system();
    asm volatile("st.release.sys.u32 [%0], %1;" :: "l"(p), "r"(frames) : "memory");
}
// generic-proxy global stores (the plane histories) -> visible to later bulk copies (async proxy) once a barrier orders them
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ---- split-fp16 plane histories (DecParams::pl_hist, numerics.cuh) ------------------------------------------------------
// index (in halfs) of channel c of row t of utterance b in the hi plane; the lo plane follows at + 2 * rows * 8
__device__ __forceinline__ size_t pl_idx(int nslab, int rows, int b, int c, int t) {
    return ((size_t)(b * nslab + (c >> 4)) * 4 + ((c >> 3) & 1)) * (size_t)rows * 8 + (size_t)(t + DEC_PL_PAD) * 8 + (c & 7);
}
// two independent fp32 FMAs on (x, y) pairs
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ uint64_t* bar64(unsigned long long* p) { return reinterpret_cast<uint64_t*>(p); }

// ---- the virtual weight stream ---------------------------------------------------------------------
// frame f = AudioEnc chunks, [the AudioDec chunks of the receptive-field blocks, if a window moved in f], AudioDec chunks
struct Cur { int f, seg, c; };
__device__ __forceinline__ void cur_next(const DecParams& P, const Smem& S, Cur& u) {
    u.c++;
    const int end = (u.seg == 0) ? P.nch_enc : (u.seg == 1 ? P.pyr_ch1 : P.nch);
    if (u.c < end) return;
    if (u.seg == 0) {
        if (S.fmoved[u.f & 1]) { u.seg = 1; u.c = P.pyr_ch0; } else { u.seg = 2; u.c = P.nch_enc; }
    } else if (u.seg == 1) { u.seg = 2; u.c = P.nch_enc; }
    else { u.f++; u.seg = 0; u.c = 0; }
}
struct Stream {
    const float* base;          // this rank's packed stream
    Cur prod;                   // chunk that will be loaded into the slot the consumer frees next (the consumer itself walks the blocks' chunk ranges)
    unsigned pos;               // number of chunks consumed so far
    unsigned tcq;               // pre-pass: slabs staged so far (mbarrier phase parities)
};
// one lane of warp `warp`: load the warp's rows of chunk `u` into its region of `slot`.  STOP: the cluster executes S.f_end
// frames; S.f_end is lowered at a frame's attention, before the AudioDec refills that carry the cursor into the next frame,
// so no copy of a frame that will not run is ever issued and none is in flight when the cluster exits.
template <bool STOP>
__device__ __forceinline__ void stream_issue(const DecParams& P, Smem& S, const Stream& st, const Cur& u, int slot, int warp) {
    if (u.f >= (STOP ? S.f_end : P.steps)) return;
    const DecChunk& ch = P.C[u.c];
    const uint32_t bytes = (uint32_t)ch.nfl4 * 2u;                   // nfl * 4 bytes / 8 warps
    mbar_expect_tx(bar64(&S.fullw[slot][warp]), bytes);
    const int off = (u.seg == 1) ? ch.off16 : ch.off;                // the pre-pass reads the same rows as split-fp16 MMA slabs
    bulk_g2s(&S.ring[slot][warp][0], st.base + off + warp * (ch.nfl4 >> 1), bytes, &S.fullw[slot][warp]);
}
__device__ __forceinline__ void stream_advance(const DecParams& P, const Smem& S, Stream& st) {
    cur_next(P, S, st.prod); st.pos++;
}
// the calling warp has read its region of the current chunk: refill it with its rows of the chunk 3 ahead
template <bool STOP>
__device__ __forceinline__ void warp_release(const DecParams& P, Smem& S, Stream& st, int warp, int lane) {
    __syncwarp();                                                     // every lane's loads of the region have returned (their FMAs have issued)
    if (lane == 0) stream_issue<STOP>(P, S, st, st.prod, (int)(st.pos % DEC_NSLOT), warp);
    stream_advance(P, S, st);
}

// ---- prefetch of the next block's parameters and dilated taps -------------------------------------------
__device__ __forceinline__ void prefetch_params(const DecParams& P, Smem& S, int li, int rank) {
    const DecLayer& l = P.L[li];
    float* dst = S.prm[li & 1];
    const int tid = threadIdx.x;
    cp_async16(dst + tid * 4, P.lnp[li] + tid * 4, true);                        // 1024 floats
    // bias slice in stream column order -- hc: columns [0,cs) gate of channels rank*cs.., [cs,2cs) info; conv: [0,cs), zero beyond
    if ((l.cs & 3) == 0) {
        if (tid < l.ns / 4) {
            const int n = tid * 4;
            cp_async16(dst + 1024 + n, P.bias[li] + ((l.kind == 1 && n >= l.cs) ? l.cout + rank * l.cs + (n - l.cs) : rank * l.cs + n), true);
        }
    } else if (tid < l.ns) {                                                     // the n_mels-wide last block (5 channels per CTA)
        dst[1024 + tid] = (tid < l.cs) ? __ldg(P.bias[li] + rank * l.cs + tid) : 0.f;
    }
}
// taps (all but the last) of block li at frame j: rows j - (ntaps-1-tap)*rate of its input history -> xin[buf][g][tap*256..]
// (multi-tap blocks have 256 input channels and 3 taps: decode_tables checks it)
__device__ __forceinline__ void prefetch_taps(const DecParams& P, Smem& S, int li, int j, int b0, int G, int buf) {
    const DecLayer& l = P.L[li];
    if (l.ntaps != 3 || !P.in_hist[li]) return;
    for (int i = threadIdx.x; i < G * 128; i += NT) {
        const int c4 = i & 63, tap = (i >> 6) & 1, g = i >> 7;
        const int t = j - (2 - tap) * l.rate;
        const float* src = P.in_hist[li] + ((size_t)(b0 + g) * P.T + (t < 0 ? 0 : t)) * 256 + c4 * 4;
        cp_async16(&S.xin[buf][g][tap * 256 + c4 * 4], src, t >= 0);
    }
}

// ---- GEMV of the calling warp's k rows of one chunk: acc[g] += sum_k x[g][k] * W[k][n] ----------------------
// wreg: the warp's region ([k/4][column][4]); x: row 0 of the input vectors at the warp's first k; ns = 32 / 16 / 8 columns
// per CTA.  The utterance count GT is a template parameter of the whole kernel (only ONE instantiation runs per launch, so the
// instruction-cache footprint is that of one): no per-utterance branches, all loads of an 8-k step hoisted, two independent
// FMA chains per utterance.  Slots g >= the cluster's real utterance count multiply zeros (their input rows stay zero).
template <int GT>
__device__ __forceinline__ void gemv_warp(const float* __restrict__ wreg, const float* __restrict__ x, int kr8, int ns, float (&acc)[GT]) {
    const int lane = threadIdx.x & 31;
    const int lg = (ns == 32) ? 5 : (ns == 16 ? 4 : 3);
    const int n = lane & (ns - 1), sg = lane >> lg;                  // column, k sub-group inside the warp
    const int kper = kr8 >> (5 - lg);                                // k rows per sub-group, multiple of 8
    const float* w = wreg + ((size_t)((sg * kper) >> 2) * ns + n) * 4;
    const float* xs = x + sg * kper;
    const int wstep = ns * 4;
    // Four partial sums per utterance (k mod 4 = {0,1} and {2,3} of either float4), added at the end: independent FMA chains.
    float2 p0[GT], p1[GT];
#pragma unroll
    for (int g = 0; g < GT; ++g) { p0[g] = make_float2(acc[g], 0.f); p1[g] = make_float2(0.f, 0.f); }
#pragma unroll 2
    for (int k = 0; k < kper; k += 8) {
        const float4 w0 = *reinterpret_cast<const float4*>(w);
        const float4 w1 = *reinterpret_cast<const float4*>(w + wstep);
        w += 2 * wstep;
#pragma unroll
        for (int g = 0; g < GT; ++g) {
            const float4 x0 = *reinterpret_cast<const float4*>(xs + g * XLD + k);
            const float4 x1 = *reinterpret_cast<const float4*>(xs + g * XLD + k + 4);
            float2 a = p0[g], c = p1[g];
            a = ffma2(make_float2(x0.x, x0.y), make_float2(w0.x, w0.y), a);
            c = ffma2(make_float2(x1.x, x1.y), make_float2(w1.x, w1.y), c);
            a = ffma2(make_float2(x0.z, x0.w), make_float2(w0.z, w0.w), a);
            c = ffma2(make_float2(x1.z, x1.w), make_float2(w1.z, w1.w), c);
            p0[g] = a; p1[g] = c;
        }
    }
#pragma unroll
    for (int g = 0; g < GT; ++g) acc[g] = (p0[g].x + p0[g].y) + (p1[g].x + p1[g].y);
}


// ---- the same for the 32-column slices (all hc blocks: 16 of the 24) in the PAIR-SPLIT layout ------------------------------
// The loop above is bound by shared-memory wavefronts: per 8 k a warp reads 8 wavefronts of weights and 2 x GT broadcast
// loads of the activations (every lane wants the same 8 k of x).  Here a lane owns TWO columns (2cp, 2cp+1) and HALF of the k
// (kh = lane >> 4 takes k-group 2j + kh), so a step needs ONE activation load per utterance (two addresses per warp, one
// wavefront) for the same number of FMAs: 8 + GT wavefronts instead of 8 + 2 GT.  Weight layout per 8-k block (1 KB, kernels_pack.cu):
// [column parity][k-group kh][column pair cp][4 k], so both weight loads of a warp are 512 contiguous bytes.  Partial sums of
// the two k-halves are added with one shuffle per accumulator after the last chunk.
template <int GT>
__device__ __forceinline__ void gemv_warp32(const float* __restrict__ wreg, const float* __restrict__ x, int kr8, float2 (&pe)[GT],
                                            float2 (&po)[GT]) {
    const int lane = threadIdx.x & 31, cp = lane & 15, kh = lane >> 4;
    const float* w = wreg + (kh * 16 + cp) * 4;
    const float* xs = x + kh * 4;
#pragma unroll 2
    for (int k = 0; k < kr8; k += 8) {
        const float4 wa = *reinterpret_cast<const float4*>(w);
        const float4 wb = *reinterpret_cast<const float4*>(w + 128);
        w += 256;
#pragma unroll
        for (int g = 0; g < GT; ++g) {
            const float4 xv = *reinterpret_cast<const float4*>(xs + g * XLD + k);
            float2 a = pe[g], c = po[g];
            a = ffma2(make_float2(xv.x, xv.y), make_float2(wa.x, wa.y), a);
            c = ffma2(make_float2(xv.x, xv.y), make_float2(wb.x, wb.y), c);
            a = ffma2(make_float2(xv.z, xv.w), make_float2(wa.z, wa.w), a);
            c = ffma2(make_float2(xv.z, xv.w), make_float2(wb.z, wb.w), c);
            pe[g] = a; po[g] = c;
        }
    }
}


// ---- one block on ONE row per utterance -------------------------------------------------------------------
// in: S.xin[cb][g] = [taps | current row] of the block's input, S.prm[li&1] = its parameters (both prefetched).
// out: S.xin[cb^1][g][next_off ..] = the block's output row; this CTA's channel slice appended to the output history.
template <bool PROF, int GT, bool STOP>
__device__ __forceinline__ int layer_row(const DecParams& P, Smem& S, Stream& st, int li, int j, int b0, int G, int rank, int cb, unsigned& lcount) {
    const DecLayer& l = P.L[li];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool last = (li + 1 == P.nl);
    const int nl_next = last ? 0 : li + 1;
    const int pb = (int)(lcount & 1u);
    const uint32_t gpar = (lcount >> 1) & 1u;
    const int nh = l.kind + 1;                                      // LayerNorm halves (hc: gate, info)
    // bytes every rank sends to every rank: its pre-LN slice, and a (mean, M2) LayerNorm partial per (utterance, half)
    const uint32_t gbytes = (uint32_t)(GT * l.ns * 4), pbytes = (uint32_t)(GT * nh * 8);

    cp_async_wait<0>();                     // this block's taps and parameters (issued during the previous block)
    __syncthreads();                        // barrier 1: every warp has finished the previous block (its mix wrote our input)
    if (tid == 0) mbar_expect_tx(bar64(&S.gbar[pb]), NC * (gbytes + pbytes));
    LAP(LP_START);

    if (l.ns == 32) {
        float2 pe[GT], po[GT];
#pragma unroll
        for (int g = 0; g < GT; ++g) { pe[g] = make_float2(0.f, 0.f); po[g] = make_float2(0.f, 0.f); }
        for (int c = 0; c < l.nch; ++c) {
            const DecChunk& ch = P.C[l.ch0 + c];
            const int slot = (int)(st.pos % DEC_NSLOT);
            mbar_wait(bar64(&S.fullw[slot][warp]), (st.pos / DEC_NSLOT) & 1u);
            LAP(LP_WAIT);
            const int kr8 = ch.krows >> 3;
            gemv_warp32<GT>(&S.ring[slot][warp][0], &S.xin[cb][0][ch.k0 + warp * kr8], kr8, pe, po);
            LAP(LP_GEMV);
            warp_release<STOP>(P, S, st, warp, lane);
            LAP(LP_RELEASE);
        }
#pragma unroll
        for (int g = 0; g < GT; ++g) {                              // the two k-halves of the warp (lanes l and l ^ 16)
            float e = pe[g].x + pe[g].y, o = po[g].x + po[g].y;
            e += __shfl_xor_sync(0xffffffffu, e, 16);
            o += __shfl_xor_sync(0xffffffffu, o, 16);
            if (lane < 16) *reinterpret_cast<float2*>(&S.red[g][warp * 32 + 2 * lane]) = make_float2(e, o);
        }
    } else {
        float acc[GT];
#pragma unroll
        for (int g = 0; g < GT; ++g) acc[g] = 0.f;
        for (int c = 0; c < l.nch; ++c) {
            const DecChunk& ch = P.C[l.ch0 + c];
            const int slot = (int)(st.pos % DEC_NSLOT);
            mbar_wait(bar64(&S.fullw[slot][warp]), (st.pos / DEC_NSLOT) & 1u);
            LAP(LP_WAIT);
            const int kr8 = ch.krows >> 3;
            gemv_warp<GT>(&S.ring[slot][warp][0], &S.xin[cb][0][ch.k0 + warp * kr8], kr8, l.ns, acc);
            LAP(LP_GEMV);
            warp_release<STOP>(P, S, st, warp, lane);
            LAP(LP_RELEASE);
        }
#pragma unroll
        for (int g = 0; g < GT; ++g) S.red[g][tid] = acc[g];
    }
    __syncthreads();                        // barrier 2: every warp's partial sums are in S.red
    // All-gather from registers: thread (g, n) finishes value n of utterance g of the slice (same order as always: bias, even
    // and odd warp partials, their sum), and the slice goes to every rank's S.pre[pb][rank] with st.async, four consecutive
    // columns per store, completing on that rank's gbar[pb].  With it, each LayerNorm half of the slice (16 channels in 16
    // consecutive lanes; 5 channels in 8 lanes for the n_mels-wide last block) ships its own statistics, pivoted on its first
    // channel: mean m_r and M2_r = sum (x - m_r)^2, computed as sum d^2 - (sum d) m' with d = x - pivot, m' = mean d.
    //
    // Reuse of S.pre[pb] / S.part[pb] (pb = block count mod 2): a rank stores block l + 2's slice only after the GEMV of
    // l + 2, which needs block l + 1's output, i.e. after its gbar wait of block l + 1, which needs OUR slice of l + 1; we
    // send that only past barrier 1 of l + 1, which every one of our threads reaches after its last read of block l's
    // values and partials (statistics merge and mix).  So nothing of l + 2 lands while block l is read.
    // gbar[pb] parity: the phase of block l completes with our arrive (expect_tx, past barrier 1 of l) and all 16 slices of
    // l.  A rank's bytes of l + 2 may land before our arrive of l + 2 (the tx count goes negative, the phase cannot complete
    // without the arrive) but not before the phase of l has completed: they follow our slice of l + 1, which we send after
    // our gbar wait of l.  Each phase therefore counts exactly one block's bytes, and the wait parity is (count / 2) & 1.
    const int lgns = (l.ns == 32) ? 5 : (l.ns == 16 ? 4 : 3);
    const int cs = l.cs;
    {
        const int nvals = GT << lgns, ng = NT >> lgns;
        if ((tid & ~31) < nvals) {                                   // warp-uniform: the shuffles below need whole warps
            const int g = tid >> lgns, n = tid & (l.ns - 1);
            float v = 0.f;
            if (tid < nvals) {
                const float* bs = S.prm[li & 1] + 1024;
                const float* rp = &S.red[g][n];
                float s0 = bs[n], s1 = 0.f;
#pragma unroll 4
                for (int q = 0; q < ng; q += 2) { s0 += rp[q << lgns]; s1 += rp[(q + 1) << lgns]; }
                v = s0 + s1;
            }
            const int W = (l.ns == 8) ? 8 : 16, w = lane & (W - 1);  // lanes of one (utterance, half); w = its column
            const float piv = __shfl_sync(0xffffffffu, v, lane & ~(W - 1));
            const float d = (w < cs) ? v - piv : 0.f;                // a constant half gives d = 0: mean = pivot, M2 = 0 exactly
            float s1 = d, s2 = d * d;
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
            if (W == 16) { s1 += __shfl_xor_sync(0xffffffffu, s1, 8); s2 += __shfl_xor_sync(0xffffffffu, s2, 8); }
            const float md = s1 * ((cs == 16) ? (1.0f / 16.0f) : __frcp_rn((float)cs));
            const float mr = piv + md, m2 = fmaxf(fmaf(-s1, md, s2), 0.f);
            const int q0 = lane & ~3;
            const float4 v4 = make_float4(__shfl_sync(0xffffffffu, v, q0), __shfl_sync(0xffffffffu, v, q0 + 1),
                                          __shfl_sync(0xffffffffu, v, q0 + 2), __shfl_sync(0xffffffffu, v, q0 + 3));
            if (tid < nvals) {
                const uint32_t bar = smem_u32(&S.gbar[pb]);
                const uint32_t vdst = smem_u32(&S.pre[pb][rank][(g << lgns) + (n & ~3)]);
                const int hf = (l.ns == 32) ? (n >> 4) : 0;
                const uint32_t pdst = smem_u32(&S.part[pb][2 * g + hf][2 * rank]);
                // the 4 lanes of a quad hold the same 4 values: each stores them to 4 of the 16 ranks
#pragma unroll
                for (int i = 0; i < NC / 4; ++i) {
                    const uint32_t r = (uint32_t)((lane & 3) + 4 * i);
                    st_async_v4(mapa(vdst, r), v4, mapa(bar, r));
                }
                for (int r = w; r < NC; r += W) st_async_v2(mapa(pdst, (uint32_t)r), mr, m2, mapa(bar, (uint32_t)r));
            }
        }
    }
    LAP(LP_GATHER);
    // prefetch for the following block, issued while the peers' slices are in flight: its taps are rows of earlier frames,
    // already in the history.  prm[nl_next & 1] was last read by the previous block's mix, and the taps go to xin[cb^1][g][0,
    // 512), which this block's mix does not write (it writes from next_off on) and nobody reads before barrier 1 of the next block.
    if (!last || j + 1 < P.steps) {
        prefetch_params(P, S, nl_next, rank);
        // the following block's input vector lives in xin[cb^1]; the attention writes the whole AudioDec C_1 input itself
        if (nl_next != P.n_enc) prefetch_taps(P, S, nl_next, last ? j + 1 : j, b0, G, cb ^ 1);
    }
    cp_async_commit();
    LAP(LP_PREFETCH);
    mbar_wait_cluster(bar64(&S.gbar[pb]), gpar);
    LAP(LP_CBAR);
    // LayerNorm statistics from the 16 ranks' partials (Chan's merge, every rank having the same cs channels of a half):
    // mean = m_0 + sum_r (m_r - m_0) / 16, M2 = sum_r M2_r + cs sum_r (m_r - mean)^2.  Relative to rank 0's mean, so equal
    // partial means -- a constant row -- give exactly zero variance (quirk Q4).  Lane 2g + hf of EVERY warp merges (g, hf) and
    // the warp's lanes read the results by shuffle: no block barrier.  Then gate / highway mix one thread per channel.
    // Redundantly in every CTA: the next block's input is local.
    {
        const int C = l.cout;
        const float rC = (C == 256) ? (1.0f / 256.0f) : __frcp_rn((float)C);
        float mu = 0.f, rs = 0.f;
        if (lane < 2 * GT && (lane & 1) < nh) {
            const float* pp = &S.part[pb][lane][0];
            float4 a[NC / 2];                                         // (m, M2) of ranks 2i and 2i + 1
#pragma unroll
            for (int i = 0; i < NC / 2; ++i) a[i] = *reinterpret_cast<const float4*>(pp + 4 * i);
            const float m0 = a[0].x;
            float sd0 = 0.f, sd1 = 0.f;                               // even and odd ranks: two independent chains
#pragma unroll
            for (int i = 0; i < NC / 2; ++i) { sd0 += a[i].x - m0; sd1 += a[i].z - m0; }
            mu = m0 + (sd0 + sd1) * (1.0f / NC);
            float q0 = 0.f, q1 = 0.f, e0 = 0.f, e1 = 0.f;
#pragma unroll
            for (int i = 0; i < NC / 2; ++i) {
                const float d0 = a[i].x - mu, d1 = a[i].z - mu;
                q0 += a[i].y; q1 += a[i].w;
                e0 = fmaf(d0, d0, e0); e1 = fmaf(d1, d1, e1);
            }
            rs = rsqrtf(fmaxf(fmaf((float)cs, e0 + e1, q0 + q1) * rC, 0.f) + 1e-12f);
        }
        float mean[GT][2], rstd[GT][2];
#pragma unroll
        for (int g = 0; g < GT; ++g)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                mean[g][hf] = __shfl_sync(0xffffffffu, mu, 2 * g + hf);
                rstd[g][hf] = __shfl_sync(0xffffffffu, rs, 2 * g + hf);
            }
        LAP(LP_LN);
        // channel c lives in the slice of rank c / cs at column c % cs (cs = 16, or 5 for the n_mels-wide last block)
        auto pre_off = [&](int c) { const int rk = (cs == 16) ? (c >> 4) : ((c * 205) >> 10); return rk * PLD + (c - rk * cs); };
        const float* prm = S.prm[li & 1];
        const int cur_off = (l.ntaps - 1) * 256;
        const int next_off = (last || li + 1 == P.n_enc) ? 0 : (P.L[li + 1].ntaps - 1) * 256;
        float* oh = P.out_hist[li];
        __half* pl = last ? nullptr : P.pl_hist[li + 1];             // the same row as split-fp16 planes (this CTA's slice = one slab)
        const int c = tid;
        if (c < C) {
            const int po = pre_off(c);
            const bool mine = (po / PLD == rank) && oh;
            const size_t pl_lo = (size_t)P.pl_rows * 16;
            const float g1 = prm[c], b1 = prm[256 + c], g2 = prm[512 + c], b2 = prm[768 + c];
            float o[GT];
#pragma unroll
            for (int g = 0; g < GT; ++g) {
                const float* pr = &S.pre[pb][0][g << lgns];
                o[g] = (pr[po] - mean[g][0]) * rstd[g][0] * g1 + b1;
            }
            if (l.kind == 1) {
#pragma unroll
                for (int g = 0; g < GT; ++g) {
                    const float* pr = &S.pre[pb][0][g << lgns];
                    const float h2 = (pr[po + cs] - mean[g][1]) * rstd[g][1] * g2 + b2;
                    const float h1 = sigmoid_fast(o[g]);
                    o[g] = h1 * h2 + (1.0f - h1) * S.xin[cb][g][cur_off + c];
                }
            } else if (l.act == 1) {
#pragma unroll
                for (int g = 0; g < GT; ++g) o[g] = fmaxf(o[g], 0.f);
            }
#pragma unroll
            for (int g = 0; g < GT; ++g) {
                const size_t row = (size_t)(b0 + g) * P.T + j;
                if (mine && g < G) {                                  // this CTA's slice of the history row
                    oh[row * C + c] = o[g];
                    if (pl) {
                        const size_t ix = pl_idx(C >> 4, P.pl_rows, b0 + g, c, j);
                        split_f16(o[g], pl[ix], pl[ix + pl_lo]);
                    }
                }
                if (last) {                                           // Y = sigmoid(logits), networks.py:210; next frame's AudioEnc input
                    o[g] = sigmoid_fast(o[g]);
                    if (rank == 0 && g < G) P.ybuf[row * C + c] = o[g];
                }
                S.xin[cb ^ 1][g][next_off + c] = (g < G) ? o[g] : 0.f;   // unused slots stay zero
            }
        } else if (last && c < 128) {                                 // AudioEnc C_1 reads K = 128 padded channels
#pragma unroll
            for (int g = 0; g < GT; ++g) S.xin[cb ^ 1][g][c] = 0.f;
        }
    }
    LAP(LP_MIX);
    lcount++;
    return cb ^ 1;
}

// ---- attention of ONE query row under the 3-key window (networks.py:140-153) -------------------------------
// lane holds q[lane*8 .. +8); returns ctx[8] in the same layout and the argmax key (first index among equal maxima)
__device__ __forceinline__ int attend_row(const DecParams& P, const float (&qv)[8], int b, int p, int lane, float (&ctx)[8]) {
    const int d = P.d;
    const int n_lo = min(max(p, 0), P.N - 1), n_hi = min(n_lo + P.win_size, P.N);
    const float scale = rsqrtf((float)d);
    float sc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n_lo + i;
        if (n < n_hi) {
            const float* k = P.kv + ((size_t)b * P.N + n) * (2 * d) + lane * 8;
            const float4 k0 = ldcg4(k), k1 = ldcg4(k + 4);
            float s = 0.f;
            s = fmaf(qv[0], k0.x, s); s = fmaf(qv[1], k0.y, s); s = fmaf(qv[2], k0.z, s); s = fmaf(qv[3], k0.w, s);
            s = fmaf(qv[4], k1.x, s); s = fmaf(qv[5], k1.y, s); s = fmaf(qv[6], k1.z, s); s = fmaf(qv[7], k1.w, s);
            sc[i] = warp_sum(s) * scale;
        }
    }
    const int cnt = n_hi - n_lo;
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 4; ++i) if (i < cnt) mx = fmaxf(mx, sc[i]);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) if (i < cnt) { sc[i] = expf(sc[i] - mx); sum += sc[i]; }
    float best = -1.f; int besti = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) if (i < cnt) { sc[i] = sc[i] / sum; if (sc[i] > best) { best = sc[i]; besti = i; } }
#pragma unroll
    for (int i = 0; i < 8; ++i) ctx[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n_lo + i;
        if (n < n_hi) {
            const float* v = P.kv + ((size_t)b * P.N + n) * (2 * d) + d + lane * 8;
            const float4 v0 = ldcg4(v), v1 = ldcg4(v + 4);
            const float p_ = sc[i];
            ctx[0] = fmaf(p_, v0.x, ctx[0]); ctx[1] = fmaf(p_, v0.y, ctx[1]); ctx[2] = fmaf(p_, v0.z, ctx[2]); ctx[3] = fmaf(p_, v0.w, ctx[3]);
            ctx[4] = fmaf(p_, v1.x, ctx[4]); ctx[5] = fmaf(p_, v1.y, ctx[5]); ctx[6] = fmaf(p_, v1.z, ctx[6]); ctx[7] = fmaf(p_, v1.w, ctx[7]);
        }
    }
    return n_lo + besti;
}

// ---- pre-pass: refresh the receptive field (rows t < j) of the utterances whose window moved -------------------
// every moved utterance refreshes the SAME rows t_lo .. j-1 (t_lo depends on the block and the frame only), so the row list is
// (bit mask of moved utterances, first row, rows per utterance): no local arrays (see the note on the stack above)
struct PreRows { unsigned mask; int t_lo, n, total; };
__device__ __forceinline__ PreRows pre_rows(const Smem& S, int G, int j, int prow) {
    PreRows r;
    r.mask = 0;
#pragma unroll
    for (int g = 0; g < GMAX; ++g) if (g < G && S.moved[g]) r.mask |= 1u << g;
    r.t_lo = max(0, j - (prow - 1));
    r.n = j - r.t_lo;
    r.total = r.n * __popc(r.mask);
    return r;
}
// scratch row m -> (utterance, time row): the k-th moved utterance owns rows [k*n, (k+1)*n)
__device__ __forceinline__ void pre_row_of(const PreRows& r, int m, int& g, int& t) {
    const int k = m / r.n;
    unsigned mk = r.mask;
    for (int i = 0; i < k; ++i) mk &= mk - 1;                        // drop the k lowest set bits
    g = __ffs(mk) - 1;
    t = r.t_lo + (m - k * r.n);
}
__device__ __forceinline__ int pre_off_of(const PreRows& r, int g) { return r.n * __popc(r.mask & ((1u << g) - 1u)); }
// address of W[k][n] (k = row within the layer's K) inside the ring; the layer's chunks occupy consecutive slots from pos0
// ---- the pre-pass GEMM on the tensor cores (wgmma) ---------------------------------------------------------------------
// One utterance, <= TC_RA source rows.  A = the source rows as split-fp16 planes (hi = fp16(x), lo = fp16(x - hi)), staged per
// 16-channel slab in the NO-SWIZZLE K-major core-matrix layout [k8][row][8 halfs]: rows are consecutive 16-byte chunks, so
// the three taps of the dilated conv are the SAME slab read through descriptors whose start address is shifted by
// tap * rate rows -- staged once, multiplied three times.  B = this CTA's weight columns, pre-packed in the same layout
// ([plane][k8][column][8 halfs], 2 KB per 16-k slab) and streamed through the ring like the fp32 weights.  D = 128 x ns fp32
// in the registers of warpgroup 1 (the M = 64 halves that hold output rows); per slab and tap hi*Whi + hi*Wlo + lo*Whi (the
// dropped lo*lo term is 2^-22 relative).  The planes are kept in HBM in the same layout (pl_hist, pl_c1), so staging a slab
// is four bulk copies -- no conversion on the way.

// (descriptor start-address field, i.e. address >> 4) of every weight slab of block li, tap-major: S.tc_baddr[tap * nslab + ks].
// One division chain per entry, computed by 96 threads in parallel, OFF the MMA issue path.
__device__ __forceinline__ void pyr_tc_table(const DecParams& P, Smem& S, int li, unsigned pos0) {
    const DecLayer& l = P.L[li];
    const int nslab = l.cin / 16, spc = l.krows / 16, spr = spc / 8, slab_f = 16 * l.ns;
    const int sid = (int)threadIdx.x;
    if (sid < l.ntaps * nslab) {
        const int c = sid / spc, wi = sid - c * spc, reg = wi / spr, jj = wi - reg * spr;
        S.tc_baddr[sid] = (smem_u32(&S.ring[(pos0 + c) % DEC_NSLOT][reg][jj * slab_f]) & 0x3FFFFu) >> 4;
    }
}

// warpgroup 1: the MMAs of every slab and tap into acc[row half], then the scaled, biased rows -> scratch.
// The shape is compile-time -- NS weight columns, NTAPS taps, MH live row halves of 64 (MH = 1 when every output row is below
// 64: the other half would multiply rows that are thrown away) -- so that the products of one slab are ONE straight
// fence -> MMAs -> commit sequence.  (With a run-time tap loop ptxas serialised every wgmma: C7520.)  One slab stays in
// flight: slab ks is issued before the wait for slab ks - 1, whose stage is released only after that wait.  Slabs are
// numbered through the launch from q0 (see pyr_tc_utt); the release of slab q goes to the CTA that stages slab q + TC_NSTG.
// A layout of a stage: PACKED = false, one utterance's window of source rows, tap t read from row t * rate of it;
// PACKED = true, one image per tap of the rows that tap reads for all moved utterances (pyr_tc_packed).
template <bool PROF, int NS, int NTAPS, int MH, bool PACKED>
__device__ __forceinline__ void pyr_mma_rows(const DecParams& P, Smem& S, int li, unsigned q0, int n_out, int rank,
                                             float* scr_rows) {
    const DecLayer& l = P.L[li];
    const int nslab = l.cin / 16, lane = threadIdx.x & 31, w4 = (threadIdx.x >> 5) & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    long long t_prof = 0;                                             // lap timers of this warpgroup (thread 128)
    auto wlap = [&](int i) {
        if constexpr (PROF) { if (leader) { const long long now = clock64(); if (i >= 0) S.prof[i] += now - t_prof; t_prof = now; } }
    };
    wlap(-1);
    unsigned char* As = &S.tca[0][0];
    const uint64_t dA0 = gmma_desc_noswz(0, (PACKED ? TC_PR : TC_RA) * 16, 128), dB0 = gmma_desc_noswz(0, (uint32_t)NS * 16, 128);
    const uint32_t a_base = (smem_u32(As) & 0x3FFFFu) >> 4, b_lo = (uint32_t)NS * 2;
    const uint32_t tap_step = PACKED ? (uint32_t)(TC_PTAP >> 4) : (uint32_t)l.rate;
    constexpr uint32_t a_lo = (PACKED ? 2 * TC_PR * 16 : TC_APLANE) >> 4;
    float acc[MH][NS / 2];
#pragma unroll
    for (int m = 0; m < MH; ++m)
#pragma unroll
        for (int i = 0; i < NS / 2; ++i) acc[m][i] = 0.f;
    auto release = [&](unsigned q) { mbar_arrive_remote(bar64(&S.sbar[q % TC_NSTG]), (q + TC_NSTG) % NC); };
    unsigned q = q0;
#pragma unroll 1
    for (int ks = 0; ks < nslab; ++ks, ++q) {
        uint32_t bt[NTAPS];
#pragma unroll
        for (int tap = 0; tap < NTAPS; ++tap) bt[tap] = S.tc_baddr[tap * nslab + ks];
        const unsigned stg = q % TC_NSTG;
        const uint32_t aa = a_base + stg * (TC_ASTAGE >> 4);
        mbar_wait(bar64(&S.abar[stg]), (q / TC_NSTG) & 1u);          // the slab is staged (its bulk copies completed)
        wlap(LP_WG_AWAIT);
        wg_fence();
#pragma unroll
        for (int tap = 0; tap < NTAPS; ++tap) {
            const uint64_t db_hi = dB0 | bt[tap], db_lo = dB0 | (bt[tap] + b_lo);
#pragma unroll
            for (int m = 0; m < MH; ++m) {                            // rows 64 m .. 64 m + 63: 64 rows of 16 bytes further
                const uint32_t a = aa + (uint32_t)tap * tap_step + 64u * m;
                const uint64_t da_hi = dA0 | a, da_lo = dA0 | (a + a_lo);
                wgmma_f16<NS / 16>(acc[m], da_hi, db_hi, (ks | tap) != 0);
                wgmma_f16<NS / 16>(acc[m], da_hi, db_lo, 1u);
                wgmma_f16<NS / 16>(acc[m], da_lo, db_hi, 1u);
            }
        }
        wg_commit();
        wg_wait<1>();                                                 // slab ks - 1 is multiplied: its stage may be refilled
        if (ks > 0 && leader) release(q - 1);
        wlap(LP_WG_MMA);
    }
    wg_wait<0>();
#pragma unroll
    for (int m = 0; m < MH; ++m) wg_fence_regs(acc[m]);
    if (leader) release(q - 1);
    wlap(LP_WG_MMA);
    const float inv = P.inv_scale[li];
    const float* bs = P.bias[li];
#pragma unroll
    for (int m = 0; m < MH; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = 64 * m + 16 * w4 + (lane >> 2) + 8 * h;
            if (row >= n_out) continue;
            float* orow = scr_rows + (size_t)row * 512;
#pragma unroll
            for (int i = 0; i < NS / 8; ++i) {
                // hc: columns [0,16) gate, [16,32) info of channels rank*16..; conv: [0,16)
                const int n = i * 8 + 2 * (lane & 3), hf = n >> 4, nn = n & 15;
                const int col = hf * 256 + rank * 16 + nn, bi = hf * l.cout + rank * 16 + nn;
                const float2 bq = __ldg(reinterpret_cast<const float2*>(bs + bi));
                *reinterpret_cast<float2*>(orow + col) = make_float2(fmaf(acc[m][i * 4 + 2 * h], inv, bq.x),
                                                                     fmaf(acc[m][i * 4 + 2 * h + 1], inv, bq.y));
            }
        }
    wlap(LP_WG_EPI);
}

// The slab pipeline has no block barrier, and every slab is fetched from L2 once per cluster: every CTA needs the whole K
// of the same source rows for its own output columns, so slab q is staged by ONE CTA, rank q % NC, with bulk copies
// multicast to the same stage of all NC CTAs, each completing on that CTA's own abar[s].  Slabs are numbered through the
// whole launch (st.tcq, the same in every CTA: the moved mask is computed identically everywhere): slab q lives in stage
// s = q % TC_NSTG and is that stage's (q / TC_NSTG)-th use, which gives every wait its phase parity without a shared counter.
//   * Thread 0 of every CTA arms abar[s] for slab q (expected bytes) once its previous slab in that stage has landed, so
//     the arming opens the right phase; the multicast may land before the arming (the transaction count then runs negative
//     until it).
//   * Stage s may be overwritten with slab q once every CTA's MMA warpgroup has multiplied slab q - TC_NSTG.  Those NC
//     releases go to sbar[s] of the CTA that stages slab q, and to no other CTA: sbar[s] of CTA r then counts releases of
//     the slabs q - TC_NSTG with q = r mod NC and q = s mod TC_NSTG only, one every TC_QCYC slabs, and the slab after
//     cannot be released before this CTA has staged the slab in between -- so no release is ever counted in the wrong
//     phase, and the phase of slab q's wait is (q - TC_NSTG) / TC_QCYC.
// Source of the slabs: the plane history of the block's input (rows t_lo - halo .. t_lo + n_out - 1 of utterance b: four
// runs of n_src rows, the zero rows in front of t = 0 included), or for the first AudioDec block the cluster's plane
// scratch of the recomputed rows, `c1` (a whole stage per slab).
template <bool PROF>
__device__ __forceinline__ void pyr_tc_utt(const DecParams& P, Smem& S, int li, unsigned q0, int b, int t_lo, int n_out,
                                        int rank, float* scr_rows, const __half* c1) {
    const DecLayer& l = P.L[li];
    const int tid = threadIdx.x, warp = tid >> 5;
    if (tid == 0) {
        const int halo = (l.ntaps - 1) * l.rate, n_src = n_out + halo;   // <= TC_RA (decode_tables)
        const int nslab = l.cin / 16;
        const size_t run = (size_t)P.pl_rows * 8;                     // halfs between the four (plane, k8) runs of a slab
        const __half* src = c1 ? c1 : P.pl_hist[li] + pl_idx(nslab, P.pl_rows, b, 0, t_lo - halo);
        const size_t sstep = c1 ? (size_t)TC_ASTAGE / 2 : 4 * run;    // halfs per slab
        const uint32_t rb = (uint32_t)n_src * 16;
        const uint16_t all = (uint16_t)((1u << NC) - 1u);
        fence_proxy_async_global();
        unsigned q = q0;
#pragma unroll 1
        for (int ks = 0; ks < nslab; ++ks, src += sstep, ++q) {
            const unsigned stg = q % TC_NSTG, use = q / TC_NSTG;
            if (use > 0) mbar_wait(bar64(&S.abar[stg]), (use - 1) & 1u);   // this CTA's previous slab in the stage has landed
            mbar_expect_tx(bar64(&S.abar[stg]), c1 ? (uint32_t)TC_ASTAGE : 4 * rb);
            if (q % NC != (unsigned)rank) continue;
            if (use > 0) mbar_wait(bar64(&S.sbar[stg]), ((q - TC_NSTG) / TC_QCYC) & 1u);   // every CTA has multiplied slab q - TC_NSTG
            unsigned char* dst = &S.tca[stg][0];
            if (c1) {
                bulk_g2s_mc(dst, src, TC_ASTAGE, &S.abar[stg], all);
            } else {
#pragma unroll
                for (int r = 0; r < 4; ++r)                           // (plane, k8 group) = (r >> 1, r & 1)
                    bulk_g2s_mc(dst + (r >> 1) * TC_APLANE + (r & 1) * (TC_RA * 16), src + r * run, rb, &S.abar[stg], all);
            }
        }
    } else if (warp >= 4) {                                           // shapes checked by decode_tables: hc 32 columns x 3 taps, conv 16 x 1
        if (l.ns == 32) {
            if (n_out > 64) pyr_mma_rows<PROF, 32, 3, 2, false>(P, S, li, q0, n_out, rank, scr_rows);
            else pyr_mma_rows<PROF, 32, 3, 1, false>(P, S, li, q0, n_out, rank, scr_rows);
        } else {
            if (n_out > 64) pyr_mma_rows<PROF, 16, 1, 2, false>(P, S, li, q0, n_out, rank, scr_rows);
            else pyr_mma_rows<PROF, 16, 1, 1, false>(P, S, li, q0, n_out, rank, scr_rows);
        }
    }
    // no block barrier: thread 0 goes on to the next utterance's slabs while this one's rows are stored (the stage
    // mbarriers order them); the caller synchronises once after the block's last utterance
}

// The short blocks (n <= 4 refreshed rows per utterance: HC_5, HC_6) as ONE M = 64 tile for all moved utterances of the
// frame: tile row m = k * n + i is row i of the k-th moved utterance, which is also its scratch row.  A dilated tap of a
// window would need the whole 2 * rate + n row window per utterance, so each slab is staged as one image per tap instead,
// holding only the rows that tap reads ([tap][plane][k8 group][TC_PR rows][8 halfs]; rows t_lo - halo + tap * rate ..
// + n - 1 of every moved utterance).  Every tile row sees the same k sequence on the same bytes as in its own tile, and
// rows >= k * n are thrown away.  Staging, multicast and release as in pyr_tc_utt.
template <bool PROF>
__device__ __forceinline__ void pyr_tc_packed(const DecParams& P, Smem& S, int li, unsigned q0, int b0, const PreRows& rl,
                                           int rank, float* scr) {
    const DecLayer& l = P.L[li];
    const int tid = threadIdx.x, warp = tid >> 5;
    if (tid == 0) {
        const int halo = (l.ntaps - 1) * l.rate, nslab = l.cin / 16, nu = __popc(rl.mask);
        const size_t run = (size_t)P.pl_rows * 8;                     // halfs between the four (plane, k8) runs of a slab
        const uint32_t rb = (uint32_t)rl.n * 16;
        const uint16_t all = (uint16_t)((1u << NC) - 1u);
        fence_proxy_async_global();
        unsigned q = q0;
#pragma unroll 1
        for (int ks = 0; ks < nslab; ++ks, ++q) {
            const unsigned stg = q % TC_NSTG, use = q / TC_NSTG;
            if (use > 0) mbar_wait(bar64(&S.abar[stg]), (use - 1) & 1u);   // this CTA's previous slab in the stage has landed
            mbar_expect_tx(bar64(&S.abar[stg]), (uint32_t)(3 * 4 * nu) * rb);
            if (q % NC != (unsigned)rank) continue;
            if (use > 0) mbar_wait(bar64(&S.sbar[stg]), ((q - TC_NSTG) / TC_QCYC) & 1u);   // every CTA has multiplied slab q - TC_NSTG
            unsigned char* dst = &S.tca[stg][0];
            unsigned mk = rl.mask;
#pragma unroll 1
            for (int k = 0; k < nu; ++k, mk &= mk - 1) {
                const int g = __ffs(mk) - 1;
                const __half* src = P.pl_hist[li] + pl_idx(nslab, P.pl_rows, b0 + g, ks * 16, rl.t_lo - halo);
#pragma unroll 1
                for (int tap = 0; tap < 3; ++tap)
#pragma unroll
                    for (int r = 0; r < 4; ++r)                       // (plane, k8 group) = (r >> 1, r & 1)
                        bulk_g2s_mc(dst + tap * TC_PTAP + r * (TC_PR * 16) + k * rb, src + (size_t)tap * l.rate * 8 + r * run, rb,
                                    &S.abar[stg], all);
            }
        }
    } else if (warp >= 4) {                                           // hc blocks only (decode_tables: 32 columns x 3 taps)
        pyr_mma_rows<PROF, 32, 3, 1, true>(P, S, li, q0, rl.total, rank, scr);
    }
}

// LayerNorm / gate / highway mix of the refreshed rows: one warp per row over the whole cluster (parameters in S.red)
__device__ __forceinline__ void pyr_ln(const DecParams& P, Smem& S, int li, int b0, const PreRows& rl, int rank, const float* scr) {
    const DecLayer& l = P.L[li];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* prm = &S.red[0][0];
    const float fC = 256.f;
    for (int m = rank * NWARP + warp; m < rl.total; m += NC * NWARP) {
        int g, t; pre_row_of(rl, m, g, t);
        const float* y = scr + (size_t)m * 512;
        const size_t row = (size_t)(b0 + g) * P.T + t;
        float z[2][8];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            if (hf > l.kind) break;
            const float4 a = ldcg4(y + hf * 256 + lane * 4), b = ldcg4(y + hf * 256 + 128 + lane * 4);
            float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) s += v[i];
            const float mean = warp_sum(s) / fC;
            float qd = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) { v[i] -= mean; qd = fmaf(v[i], v[i], qd); }
            const float inv = 1.0f / sqrtf(warp_sum(qd) / fC + 1e-12f);
            const float* gam = prm + hf * 512; const float* bet = gam + 256;
#pragma unroll
            for (int i = 0; i < 8; ++i) { const int c = (i < 4 ? 0 : 128) + lane * 4 + (i & 3); z[hf][i] = v[i] * inv * gam[c] + bet[c]; }
        }
        float o[8];
        if (l.kind == 1) {
            const float* xr = P.in_hist[li] + row * l.ldin;
            const float4 a = ldcg4(xr + lane * 4), b = ldcg4(xr + 128 + lane * 4);
            const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float h1 = sigmoid_acc(z[0][i]); o[i] = h1 * z[1][i] + (1.0f - h1) * x[i]; }
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = l.act == 1 ? fmaxf(z[0][i], 0.f) : z[0][i];
        }
        float* orow = P.out_hist[li] + row * 256;
        *reinterpret_cast<float4*>(orow + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(orow + 128 + lane * 4) = make_float4(o[4], o[5], o[6], o[7]);
        if (__half* pl = P.pl_hist[li + 1]) {                        // the next block's recompute reads these rows as planes
            const size_t lo = (size_t)P.pl_rows * 16;
            __half* p = pl + pl_idx(16, P.pl_rows, b0 + g, lane * 4, t);           // four consecutive channels of one row
            split_store_f16<4>(o, p, p + lo);
            p = pl + pl_idx(16, P.pl_rows, b0 + g, 128 + lane * 4, t);
            split_store_f16<4>(o + 4, p, p + lo);
        }
    }
}

}  // namespace

// ---- the pre-pass.  Inlined: a wgmma pipeline must not cross a call boundary -- with the pre-pass out of line ptxas
// serialised every MMA in it (C7510).  The stream cursors go in and come back by value; everything else lives in shared memory.
template <bool PROF, bool STOP>
__device__ __forceinline__ Stream prepass(const DecParams& P, Smem& S, Stream st, int j, int b0, int G, int rank, float* scr,
                                          __half* c1s) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const size_t c1_utt = (size_t)(P.L[P.n_enc].cin / 16) * (TC_ASTAGE / 2);   // halfs of one utterance's C_1 planes

            // ---- pre-pass: rows t < j of the moved utterances under the new window (uniform branch: see the file header) ----
            if (threadIdx.x == 0) { S.n_moved_frames++; for (int g = 0; g < G; ++g) S.n_moved_utt += S.moved[g]; }
            const PreRows ra = pre_rows(S, G, j, P.L[P.n_enc].prow);
            const float* Qh = P.out_hist[P.n_enc - 1];
            for (int m = rank * NWARP + warp; m < ra.total; m += NC * NWARP) {
                int g, t; pre_row_of(ra, m, g, t);
                const size_t row = (size_t)(b0 + g) * P.T + t;
                float qv[8], ctx[8];
                const float4 q0 = ldcg4(Qh + row * P.d + lane * 8), q1 = ldcg4(Qh + row * P.d + lane * 8 + 4);
                qv[0] = q0.x; qv[1] = q0.y; qv[2] = q0.z; qv[3] = q0.w; qv[4] = q1.x; qv[5] = q1.y; qv[6] = q1.z; qv[7] = q1.w;
                attend_row(P, qv, b0 + g, S.p_cur[g], lane, ctx);
                float* rr = P.rbuf + row * (2 * P.d);
                *reinterpret_cast<float4*>(rr + lane * 8) = make_float4(ctx[0], ctx[1], ctx[2], ctx[3]);
                *reinterpret_cast<float4*>(rr + lane * 8 + 4) = make_float4(ctx[4], ctx[5], ctx[6], ctx[7]);
                *reinterpret_cast<float4*>(rr + P.d + lane * 8) = q0;
                *reinterpret_cast<float4*>(rr + P.d + lane * 8 + 4) = q1;
                // the same row as the first AudioDec block's A operand: slab-major planes, row t - t_lo of utterance g's stage
                // images (lane holds channels lane * 8 .. + 8 of [ctx | q]: slab lane / 2 (+ d / 16), k8 group lane % 2)
                __half* cs = c1s + (size_t)g * c1_utt + (size_t)(lane >> 1) * (TC_ASTAGE / 2) + (lane & 1) * (TC_RA * 8) + (t - ra.t_lo) * 8;
                split_store_f16<8>(ctx, cs, cs + TC_APLANE / 2);              // the lo plane: TC_APLANE bytes further
                __half* cq = cs + (size_t)(P.d >> 4) * (TC_ASTAGE / 2);
                split_store_f16<8>(qv, cq, cq + TC_APLANE / 2);
            }
            fence_proxy_async_global();                   // the plane rows are read by bulk copies after the barrier
            cluster_sync_all();
            LAP(LP_PYR_ATT);
            for (int lp = P.n_enc; lp < P.nl && P.L[lp].prow > 1; ++lp) {
                const DecLayer& l = P.L[lp];
                // every warp waits for ALL regions of the block's chunks (lane w watches region w)
                for (int c = 0; c < l.nch; ++c) {
                    const unsigned pp = st.pos + c;
                    if (lane < NWARP) mbar_wait(bar64(&S.fullw[pp % DEC_NSLOT][lane]), (pp / DEC_NSLOT) & 1u);
                }
                __syncwarp();
                LAP(LP_PYR_WTS);
                const PreRows rl = pre_rows(S, G, j, l.prow);
                if (rl.n > 0) {
                    pyr_tc_table(P, S, lp, st.pos);
                    __syncthreads();
                    LAP(LP_PYR_TABLE);
                    if (l.ns == 32 && (l.prow - 1) * GMAX <= TC_PR) {   // short block: one tile for all moved utterances
                        pyr_tc_packed<PROF>(P, S, lp, st.tcq, b0, rl, rank, scr);
                        st.tcq += l.cin / 16;
                    } else for (int g = 0; g < G; ++g) {
                        if (!((rl.mask >> g) & 1u)) continue;
                        float* rows = scr + (size_t)pre_off_of(rl, g) * 512;
                        pyr_tc_utt<PROF>(P, S, lp, st.tcq, b0 + g, rl.t_lo, rl.n, rank, rows, lp == P.n_enc ? c1s + (size_t)g * c1_utt : nullptr);
                        st.tcq += l.cin / 16;
                    }
                    LAP(LP_PYR_STAGE);
                }
                __syncthreads();                          // every warp is done with every region of these chunks
                LAP(LP_PYR_DRAIN);
                for (int c = 0; c < l.nch; ++c) {
                    if (lane == 0) { fence_proxy_async_smem(); stream_issue<STOP>(P, S, st, st.prod, (int)(st.pos % DEC_NSLOT), warp); }
                    stream_advance(P, S, st);
                }
                for (int i = tid; i < 256; i += NT)       // this block's LayerNorm parameters for pyr_ln
                    *reinterpret_cast<float4*>(&S.red[0][0] + i * 4) = __ldg(reinterpret_cast<const float4*>(P.lnp[lp]) + i);
                LAP(LP_PYR_REFILL);
                cluster_sync_all();
                LAP(LP_PYR_BAR);
                pyr_ln(P, S, lp, b0, rl, rank, scr);
                LAP(LP_PYR_LN);
                fence_proxy_async_global();               // refreshed plane rows -> the next block's bulk copies
                cluster_sync_all();
                LAP(LP_PYR_BAR);
            }
            return st;
}

// The kernel body.  STOP (decode_until_kernel): after frame j's attention every CTA applies the end-of-utterance rule to
// S.p_next -- computed identically in every CTA -- so all 16 CTAs leave the frame loop after the same frame, with no
// extra communication, and go through the ordinary epilogue.
// PATH (decode_path_kernel, with STOP): the window of frame j + 1 is path[b][j + 1] instead of the argmax of row j, which
// is only recorded in amax_hist[b][j] (both (B, T)).  The lengths are inputs (P.lengths): S.f_end, the longest of the
// cluster's, is set before the first frame and never lowered (S.stop / S.ulen are not used); the host pads each path row
// past its length with its last window, so those frames never trigger a recompute.
// PROG (decode_progress_kernel, with STOP): at the end of every frame the cluster publishes its progress to `prog`, host
// memory mapped into the device (publish_progress).
template <bool PROF, int GT, bool STOP, bool PATH = false, bool PROG = false>
__device__ __forceinline__ void decode_body(const DecParams& Pc, const int* __restrict__ path = nullptr,
                                            int* __restrict__ amax_hist = nullptr, int* prog = nullptr) {
    static_assert(!PATH || STOP, "a path decode is bounded by its lengths");
    static_assert(!PROG || (STOP && !PATH), "progress is published by the until-EOS decode");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem& S = *reinterpret_cast<Smem*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    {
        const int* src = reinterpret_cast<const int*>(&Pc);
        int* dst = reinterpret_cast<int*>(&S.P);
        for (int i = tid; i < (int)(sizeof(DecParams) / 4); i += NT) dst[i] = src[i];
    }
    __syncthreads();
    const DecParams& P = S.P;
    const int rank = (int)cluster_ctarank();
    const int cluster = blockIdx.x / NC;
    const int b0 = cluster * P.G;
    const int G = min(P.G, P.B - b0);
    float* scr = P.pre_scr + (size_t)cluster * P.G * 85 * 512;
    __half* c1s = P.pl_c1 + (size_t)cluster * P.G * (P.L[P.n_enc].cin / 16) * (TC_ASTAGE / 2);

    if (tid == 0) {
        for (int s = 0; s < DEC_NSLOT; ++s)
            for (int w = 0; w < NWARP; ++w) mbar_init(bar64(&S.fullw[s][w]), 1);
        mbar_init(bar64(&S.gbar[0]), 1); mbar_init(bar64(&S.gbar[1]), 1);
        for (int i = 0; i < TC_NSTG; ++i) { mbar_init(bar64(&S.sbar[i]), NC); mbar_init(bar64(&S.abar[i]), 1); }
        fence_mbar_init();
    }
    for (int i = tid; i < 2 * GMAX * XLD; i += NT) (&S.xin[0][0][0])[i] = 0.f;
    for (int i = tid; i < 2 * NC * PLD; i += NT) (&S.pre[0][0][0])[i] = 0.f;
    if (tid < GMAX) { S.p_cur[tid] = 0; S.p_prev[tid] = 0; S.p_next[tid] = 0; S.moved[tid] = 0; }
    if (tid < 2) S.fmoved[tid] = 0;
    if (tid < DEC_NPROF) S.prof[tid] = 0;
    if (tid == 0) { S.n_moved_frames = 0; S.n_moved_utt = 0; }
    if constexpr (PATH) {
        if (tid < GMAX) {
            const int p0 = tid < G ? path[(size_t)(b0 + tid) * P.T] : 0;
            S.p_cur[tid] = p0; S.p_prev[tid] = p0;
        }
        if (tid == 0) {
            int fe = 0;
            for (int g = 0; g < G; ++g) fe = max(fe, P.lengths[b0 + g]);
            S.f_end = fe;
        }
    } else if constexpr (STOP) {                          // slots past the cluster's utterances count as ended at frame 0
        if (tid < GMAX) { S.stop[tid] = tid < G ? P.stop_pos[b0 + tid] : -1; S.ulen[tid] = tid < G ? -1 : 0; }
        if (tid == 0) S.f_end = P.steps;
    }
    __syncthreads();

    Stream st;
    st.base = P.wstream + (size_t)rank * P.stream_len;
    st.prod = Cur{0, 0, 0}; st.pos = 0; st.tcq = 0;
    for (int s = 0; s < DEC_NSLOT; ++s) {                // the first chunks are AudioEnc chunks of frame 0 (nch_enc > DEC_NSLOT)
        if (lane == 0) stream_issue<STOP>(P, S, st, st.prod, s, warp);
        cur_next(P, S, st.prod);
    }
    prefetch_params(P, S, 0, rank);
    cp_async_commit();
    cluster_sync_all();                                   // every CTA of the cluster is running: DSMEM and its barriers exist

    int cb = 0;
    unsigned lcount = 0;
    __syncthreads();
    if (tid == 0) S.prof_last = clock64();
    int frames = P.steps;
    for (int j = 0; j < P.steps; ++j) {
        if (tid < GMAX) S.moved[tid] = (tid < G && j > 0 && (P.force_prepass || S.p_cur[tid] != S.p_prev[tid])) ? 1 : 0;
        if (tid == 0) {
            int any = 0;
            for (int g = 0; g < G; ++g) any |= (j > 0 && (P.force_prepass || S.p_cur[g] != S.p_prev[g])) ? 1 : 0;
            S.fmoved[j & 1] = any;
        }
        __syncthreads();
        const bool any_moved = S.fmoved[j & 1] != 0;
        if (rank == 0 && tid < G) P.p_hist[(size_t)(b0 + tid) * P.T + j] = S.p_cur[tid];

        // AudioEnc (networks.py:81-124; input Y[j-1], train.py:51, already in xin[cb]), Attention, AudioDec (networks.py:166-212):
        // ONE copy of the block body in the instruction stream -- the per-frame loop has to stay inside the instruction cache
        for (int li = 0; li < P.nl; ++li) {
        if (li == P.n_enc) {
        // Attention of row j under the current window, redundantly in every CTA: R[j] = [A.V ; Q] (networks.py:140-153)
        __syncthreads();                                  // Q[j] was written one thread per channel
        if (warp < G) {
            const int g = warp;
            float qv[8], ctx[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) qv[i] = S.xin[cb][g][lane * 8 + i];
            const int amax = attend_row(P, qv, b0 + g, S.p_cur[g], lane, ctx);
            if constexpr (PATH) {
                if (lane == 0) {
                    const size_t row = (size_t)(b0 + g) * P.T;
                    if (rank == 0) amax_hist[row + j] = amax;
                    S.p_next[g] = j + 1 < P.steps ? path[row + j + 1] : S.p_cur[g];
                }
            } else {
                if (lane == 0) S.p_next[g] = amax;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) { S.xin[cb ^ 1][g][lane * 8 + i] = ctx[i]; S.xin[cb ^ 1][g][P.d + lane * 8 + i] = qv[i]; }
        }
        cb ^= 1;
        LAP(LP_ATT);
        if constexpr (STOP && !PATH) {
            // argmax of row j = S.p_next.  Utterance g ends at min(steps, j + 1 + tail) once it reaches its stop position;
            // when every utterance has a length the cluster executes the longest.  S.f_end >= j + 1 here, and the refill
            // cursor is still inside frame j (the AudioDec chunks of a frame outnumber the ring slots: checked by the host),
            // so lowering the bound now keeps every chunk of frame f_end unissued.  The next block barrier (layer_row's
            // first, or the pre-pass's cluster barrier) publishes it before any refill.
            __syncthreads();
            if (tid == 0) {
                int fe = 0;
                for (int g = 0; g < GMAX; ++g) {
                    if (S.ulen[g] < 0 && S.stop[g] >= 0 && S.p_next[g] >= S.stop[g]) S.ulen[g] = min(P.steps, j + 1 + P.tail);
                    fe = (fe < 0 || S.ulen[g] < 0) ? -1 : max(fe, S.ulen[g]);
                }
                if (fe >= 0) S.f_end = fe;
            }
        }

        if (any_moved) st = prepass<PROF, STOP>(P, S, st, j, b0, G, rank, scr, c1s);
        }   // li == n_enc
        cb = layer_row<PROF, GT, STOP>(P, S, st, li, j, b0, G, rank, cb, lcount);
        }   // blocks

        __syncthreads();
        if (tid < GMAX) { S.p_prev[tid] = S.p_cur[tid]; S.p_cur[tid] = S.p_next[tid]; }
        fence_proxy_async_global();                       // this frame's plane rows: read by bulk copies in later frames
        cluster_sync_all();                               // this frame's history rows are visible to the whole cluster
        LAP(LP_FRAME);
        if constexpr (PROG) {
            if (rank == 0 && tid == 0) publish_progress(prog + (size_t)cluster * DEC_PROG_INTS, j + 1, S.ulen);
        }
        if constexpr (STOP) {                             // S.f_end is the same in every CTA: the whole cluster leaves here
            if (j + 1 >= S.f_end) { frames = j + 1; break; }
        }
    }
    if constexpr (STOP) {
        if constexpr (!PATH) if (rank == 0 && tid < G) P.lengths[b0 + tid] = S.ulen[tid] < 0 ? P.steps : S.ulen[tid];
        if (rank == 0 && tid == 0) P.frames[cluster] = frames;
    }
    if (rank == 0 && tid < G) P.p_final[b0 + tid] = S.p_cur[tid];
    if (rank == 0 && tid == 0 && P.stats) { P.stats[2 * cluster] = S.n_moved_frames; P.stats[2 * cluster + 1] = S.n_moved_utt; }
    if (PROF && P.prof && cluster == 0 && rank == 0 && tid < DEC_NPROF) P.prof[tid] = S.prof[tid];
    cp_async_wait<0>();
    cluster_sync_all();                                   // no CTA exits while a peer may still write into its shared memory
}

template <bool PROF, int GT>
__global__ void __cluster_dims__(DEC_NC, 1, 1) __launch_bounds__(DEC_THREADS, 1)
decode_cluster_kernel(const __grid_constant__ DecParams Pc) { decode_body<PROF, GT, false>(Pc); }

// the same loop ending each utterance at its text (DecParams::stop_pos); a separate kernel, so that the frame loop of
// decode_cluster_kernel is the one it always was
template <int GT>
__global__ void __cluster_dims__(DEC_NC, 1, 1) __launch_bounds__(DEC_THREADS, 1)
decode_until_kernel(const __grid_constant__ DecParams Pc) { decode_body<false, GT, true>(Pc); }

// decode_until_kernel that publishes its progress at the end of every frame: progress[cluster * DEC_PROG_INTS ...]
template <int GT>
__global__ void __cluster_dims__(DEC_NC, 1, 1) __launch_bounds__(DEC_THREADS, 1)
decode_progress_kernel(const __grid_constant__ DecParams Pc, int* progress) {
    decode_body<false, GT, true, false, true>(Pc, nullptr, nullptr, progress);
}

// the same loop along a caller's window path: path and amax_hist are (B, T), P.lengths (B) are the frames to produce
template <int GT>
__global__ void __cluster_dims__(DEC_NC, 1, 1) __launch_bounds__(DEC_THREADS, 1)
decode_path_kernel(const __grid_constant__ DecParams Pc, const int* __restrict__ path, int* __restrict__ amax_hist) {
    decode_body<false, GT, true, true>(Pc, path, amax_hist);
}

size_t decode_smem_bytes() { return sizeof(Smem) + 128; }

using DecKernel = void (*)(DecParams);
using DecPathKernel = void (*)(DecParams, const int*, int*);
using DecProgKernel = void (*)(DecParams, int*);
static DecProgKernel decode_progress_kernel_of(int G) {
    switch (G) {
        case 1: return decode_progress_kernel<1>;
        case 2: return decode_progress_kernel<2>;
        case 3: return decode_progress_kernel<3>;
        case 4: return decode_progress_kernel<4>;
        default: return decode_progress_kernel<5>;
    }
}
static DecPathKernel decode_path_kernel_of(int G) {
    switch (G) {
        case 1: return decode_path_kernel<1>;
        case 2: return decode_path_kernel<2>;
        case 3: return decode_path_kernel<3>;
        case 4: return decode_path_kernel<4>;
        default: return decode_path_kernel<5>;
    }
}
// one instantiation per (lap timers, utterances per cluster) and per utterance count with a stop; exactly one runs in a launch
static DecKernel decode_kernel_of(bool prof, int G, bool stop = false) {
    if (stop) switch (G) {
        case 1: return decode_until_kernel<1>;
        case 2: return decode_until_kernel<2>;
        case 3: return decode_until_kernel<3>;
        case 4: return decode_until_kernel<4>;
        default: return decode_until_kernel<5>;
    }
    switch (G) {
        case 1: return prof ? decode_cluster_kernel<true, 1> : decode_cluster_kernel<false, 1>;
        case 2: return prof ? decode_cluster_kernel<true, 2> : decode_cluster_kernel<false, 2>;
        case 3: return prof ? decode_cluster_kernel<true, 3> : decode_cluster_kernel<false, 3>;
        case 4: return prof ? decode_cluster_kernel<true, 4> : decode_cluster_kernel<false, 4>;
        default: return prof ? decode_cluster_kernel<true, 5> : decode_cluster_kernel<false, 5>;
    }
}
static_assert(DEC_GMAX == 5, "decode_kernel_of: one instantiation per utterance count");

static cudaError_t decode_prepare() {
    static std::atomic<bool> done[64];                    // per device: the attributes stick to the (device, function) pair
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64 && done[dev].load(std::memory_order_acquire)) return cudaSuccess;
    for (int G = 1; G <= DEC_GMAX; ++G)
        for (int v = 0; v < 5; ++v) {                     // decode_cluster_kernel without / with lap timers, decode_until_kernel,
                                                          // decode_path_kernel, decode_progress_kernel
            const void* k = v < 3 ? reinterpret_cast<const void*>(decode_kernel_of(v == 1, G, v == 2))
                          : v == 3 ? reinterpret_cast<const void*>(decode_path_kernel_of(G))
                                   : reinterpret_cast<const void*>(decode_progress_kernel_of(G));
            e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)decode_smem_bytes());
            if (e != cudaSuccess) return e;
            e = cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
            if (e != cudaSuccess) return e;
        }
    if (dev >= 0 && dev < 64) done[dev].store(true, std::memory_order_release);
    return e;
}

int decode_max_active_clusters() {
    if (decode_prepare() != cudaSuccess) { cudaGetLastError(); return 0; }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(DEC_NC); cfg.blockDim = dim3(DEC_THREADS); cfg.dynamicSmemBytes = decode_smem_bytes();
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = DEC_NC; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, decode_kernel_of(false, DEC_GMAX), &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

cudaError_t launch_decode_cluster(const DecParams& p, int n_clusters, cudaStream_t s) {
    cudaError_t e = decode_prepare();                     // per call: the attribute is per device, handles may live on several
    if (e != cudaSuccess) return e;
    if (p.G < 1 || p.G > DEC_GMAX) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_clusters * DEC_NC); cfg.blockDim = dim3(DEC_THREADS); cfg.dynamicSmemBytes = decode_smem_bytes(); cfg.stream = s;
    cfg.attrs = nullptr; cfg.numAttrs = 0;               // cluster dims are compiled in (__cluster_dims__)
    return cudaLaunchKernelEx(&cfg, decode_kernel_of(p.prof != nullptr, p.G, p.stop_pos != nullptr), p);
}

cudaError_t launch_decode_path(const DecParams& p, const int* path, int* amax_hist, int n_clusters, cudaStream_t s) {
    cudaError_t e = decode_prepare();
    if (e != cudaSuccess) return e;
    if (p.G < 1 || p.G > DEC_GMAX || !p.lengths || !p.frames || !path || !amax_hist) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_clusters * DEC_NC); cfg.blockDim = dim3(DEC_THREADS); cfg.dynamicSmemBytes = decode_smem_bytes(); cfg.stream = s;
    cfg.attrs = nullptr; cfg.numAttrs = 0;
    return cudaLaunchKernelEx(&cfg, decode_path_kernel_of(p.G), p, path, amax_hist);
}

cudaError_t launch_decode_progress(const DecParams& p, int* progress, int n_clusters, cudaStream_t s) {
    cudaError_t e = decode_prepare();
    if (e != cudaSuccess) return e;
    if (p.G < 1 || p.G > DEC_GMAX || !p.stop_pos || !p.lengths || !p.frames || !progress) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_clusters * DEC_NC); cfg.blockDim = dim3(DEC_THREADS); cfg.dynamicSmemBytes = decode_smem_bytes(); cfg.stream = s;
    cfg.attrs = nullptr; cfg.numAttrs = 0;
    return cudaLaunchKernelEx(&cfg, decode_progress_kernel_of(p.G), p, progress);
}

__global__ void until_finish_kernel(const int* __restrict__ stop_pos, int tail, int steps, int T, int n_mels,
                                    const int* __restrict__ p_hist, int derive, int* lengths, float* Y, int* prev_hist) {
    const int b = blockIdx.x;
    __shared__ int len;
    if (threadIdx.x == 0) {
        if (derive) {
            // argmax of row j = the window of frame j + 1.  The last row is not needed: reaching the stop there gives
            // min(steps, steps + tail) = steps, the length of never reaching it.
            int n = steps;
            const int sp = stop_pos[b];
            for (int j = 0; sp >= 0 && j + 1 < steps; ++j) {
                if (p_hist[(size_t)b * T + j + 1] >= sp) { n = min(steps, j + 1 + tail); break; }
            }
            lengths[b] = n;
        }
        len = lengths[b];
    }
    __syncthreads();
    if (Y)
        for (int i = len * n_mels + (int)threadIdx.x; i < T * n_mels; i += blockDim.x) Y[(size_t)b * T * n_mels + i] = 0.f;
    if (prev_hist)
        for (int t = len + (int)threadIdx.x; t < T; t += blockDim.x) prev_hist[(size_t)b * T + t] = -1;
}

void launch_until_finish(const int* stop_pos, int tail, int steps, int T, int n_mels, const int* p_hist, bool derive,
                         int* lengths, float* Y, int* prev_hist, int B, cudaStream_t s) {
    until_finish_kernel<<<B, 256, 0, s>>>(stop_pos, tail, steps, T, n_mels, p_hist, derive ? 1 : 0, lengths, Y, prev_hist);
}

}  // namespace dctts
