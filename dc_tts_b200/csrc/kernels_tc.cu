// kernels_tc.cu -- wgmma / TMA fused block kernel for sm_90a.
//
// ONE kernel per reference block (modules.py:91-141 conv1d, :143-197 hc, :199-247
// conv1d_transpose): the dilated / causal conv as an implicit GEMM on the Hopper tensor
// cores, and the whole epilogue -- bias, LayerNorm (two of them for hc), relu / sigmoid
// gate / highway mix -- applied to the accumulator tile.
//
//   grid    (ncta, tiles); a thread-block CLUSTER of `ncta` CTAs (<= 8; 16 for the 144-column instantiation, the
//           F = 2049 blocks) shares one 128-row tile and splits the output channels; LayerNorm statistics are
//           combined across the cluster through distributed shared memory (Chan's parallel mean/M2 merge).
//   warp 0  TMA producer: per k-block (BK channels of one tap) one {BK x 128 rows} box of
//           each activation plane -- the tap's time shift is just the box coordinate, and
//           TMA's out-of-bounds zero fill IS the reference's zero padding -- plus the
//           {BK x bn} box of each weight plane, swizzled, mbarrier pipelined.
//   warpgroups 1, 2  wgmma (M=64 each, N=bn: one instruction over the CTA's whole width, K=16):
//           hi*Whi + hi*Wlo + lo*Whi per k-step into fp32 register accumulators, one k-block
//           in flight while the next is issued; then each warpgroup runs the epilogue of its
//           64 rows on its accumulator fragment: LN statistics as per-thread partial sums
//           completed over the quad that holds a row, then normalise + store.
#include "kernels_tc.cuh"
#include "numerics.cuh"
#include "tc_ptx.cuh"

#include <cstdlib>
#include <stdexcept>
#include <string>

namespace dctts {

using namespace ptx;

constexpr int TC_BM = 128;
constexpr int TC_THREADS = 384;
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_AUX_BYTES = 256 /*barriers*/ + 3 * 512 * 4 /*bias,gamma,beta*/ + 128 * 16 /*this CTA's LN partials*/;
constexpr int TC_MAX_SMEM = 227 * 1024;

// Optional progress markers into host-mapped memory (survive a trapped launch): dbg[64*cta + slot].
__device__ __forceinline__ void dbg_mark(int* dbg, int slot, int v) {
    if (dbg) {
        const int cta = blockIdx.y * gridDim.x + blockIdx.x;
        if (cta < 16) { reinterpret_cast<volatile int*>(dbg)[64 * cta + slot] = v; __threadfence_system(); }
    }
}

__device__ __forceinline__ void dbg_time(int* dbg, int slot) {
    if (dbg) dbg_mark(dbg, slot, (int)(clock64() & 0x7fffffff));
}

// The epilogue works on the m64nBN accumulator fragment (tc_ptx.cuh) in registers: the thread at (warp w4 of its
// warpgroup, lane) holds rows w4 * 16 + lane / 4 (h = 0) and that + 8 (h = 1) of its warpgroup's 64, and in each 8-column
// group q the columns 8q + 2j + {0, 1}, j = lane & 3, at v[4q + 2h + {0, 1}].  A row is spread over the 4 lanes of a quad.

// Shifted sums of columns [0, n) of groups [G0, G0 + NG) of fragment row h, completed over the quad: s = their sum, m2 =
// the sum of squared deviations from their mean.  The deviations are taken about the row's first column of the range, so
// that m2 = Q - S^2 / n does not cancel.  The order of the sums depends on the column layout only, never on the tile.
template <int G0, int NG, int R>
__device__ __forceinline__ void row_stats(const float (&v)[R], int h, int j, int n, float& s, float& m2) {
    const float piv = __shfl_sync(0xffffffffu, v[4 * G0 + 2 * h], (threadIdx.x & 31) & ~3);
    float S = 0.f, Q = 0.f;
#pragma unroll
    for (int k = 0; k < NG; ++k)
#pragma unroll
        for (int e = 0; e < 2; ++e)
            if (8 * k + 2 * j + e < n) { const float d = v[4 * (G0 + k) + 2 * h + e] - piv; S += d; Q = fmaf(d, d, Q); }
#pragma unroll
    for (int m = 1; m < 4; m <<= 1) { S += __shfl_xor_sync(0xffffffffu, S, m); Q += __shfl_xor_sync(0xffffffffu, Q, m); }
    s = piv * (float)n + S;
    m2 = fmaxf(Q - S * S / (float)max(n, 1), 0.f);
}

// 4 x 4 transpose over a quad: on entry lane j holds x[k] = part j of group k, on exit x[k] = part k of group j
__device__ __forceinline__ void quad_transpose(uint32_t (&x)[4], int j) {
#pragma unroll
    for (int m = 2; m > 0; m >>= 1) {
        const bool up = (j & m) != 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (k & m) continue;
            const uint32_t r = __shfl_xor_sync(0xffffffffu, up ? x[k] : x[k ^ m], m);
            if (up) x[k] = r; else x[k ^ m] = r;
        }
    }
}

__device__ __forceinline__ uint32_t h2_bits(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }

// Groups [G0, G0 + NG) of fragment row h -> split planes, columns col0 .. col0 + 8 NG of output row `row` (stored if ok).
// Every four groups are transposed over the quad so that each lane stores 8 consecutive columns, 16 bytes per plane, and a
// quad 64 contiguous bytes.  A group at or past the row pitch is not stored; columns past C inside it hold zeros.  All lanes
// call it (the transpose shuffles), whatever their row's ok.
template <int G0, int NG, int R>
__device__ __forceinline__ void store_planes_frag(const Planes& p, size_t row, int col0, const float (&v)[R], int h, int j,
                                                  bool ok) {
    __half* hi = p.hi + row * p.ld;
    __half* lo = p.lo + row * p.ld;
#pragma unroll
    for (int k = 0; k + 4 <= NG; k += 4) {
        uint32_t xh[4], xl[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int q = G0 + k + i;
            __half2 a, b;
            split_f16x2(make_float2(v[4 * q + 2 * h], v[4 * q + 2 * h + 1]), a, b);
            xh[i] = h2_bits(a); xl[i] = h2_bits(b);
        }
        quad_transpose(xh, j);
        quad_transpose(xl, j);
        const int col = col0 + 8 * (k + j);
        if (ok && col + 8 <= p.ld) {
            *reinterpret_cast<uint4*>(hi + col) = make_uint4(xh[0], xh[1], xh[2], xh[3]);
            *reinterpret_cast<uint4*>(lo + col) = make_uint4(xl[0], xl[1], xl[2], xl[3]);
        }
    }
#pragma unroll
    for (int k = NG & ~3; k < NG; ++k) {                                  // groups past the last four: 4 bytes per plane
        const int q = G0 + k, col = col0 + 8 * k + 2 * j;
        __half2 a, b;
        split_f16x2(make_float2(v[4 * q + 2 * h], v[4 * q + 2 * h + 1]), a, b);
        if (ok && col + 2 <= p.ld) { *reinterpret_cast<__half2*>(hi + col) = a; *reinterpret_cast<__half2*>(lo + col) = b; }
    }
}

// Columns [0, n) of groups [G0, G0 + NG) of fragment row h -> fp32 row `dst` from column col0: a quad writes 8 consecutive
// floats per group, 8-byte stores where the address allows and scalar ones otherwise.  That is one 32-byte sector only
// where the row and col0 are 32-byte aligned; the networks' fp32 outputs (80 and 1025 floats per row) mostly are not,
// so there a group spans two sectors.
template <int G0, int NG, int R>
__device__ __forceinline__ void store_f32_frag(float* dst, int col0, int n, const float (&v)[R], int h, int j) {
#pragma unroll
    for (int k = 0; k < NG; ++k) {
        const int c = 8 * k + 2 * j;
        const float x0 = v[4 * (G0 + k) + 2 * h], x1 = v[4 * (G0 + k) + 2 * h + 1];
        float* d = dst + col0 + c;
        if (c + 1 < n && (reinterpret_cast<uintptr_t>(d) & 7) == 0) *reinterpret_cast<float2*>(d) = make_float2(x0, x1);
        else { if (c < n) d[0] = x0; if (c + 1 < n) d[1] = x1; }
    }
}

// Shared memory: [ring of `stages` stages] [residual / output staging tile (hc with resid_tma)] [barriers, epilogue
// vectors, LN partials]
__host__ __device__ inline int tc_ring_bytes(int stages, int stage_bytes) { return (stages * stage_bytes + 1023) & ~1023; }
// Largest cluster of an instantiation: 16 CTAs (a non-portable cluster size) for the 144-column one, whose F = 2049 conv1d
// blocks split 2049 channels over 16 x 144; 8 for the others
__host__ __device__ constexpr int tc_max_cluster(int bn) { return bn == 144 ? 16 : 8; }
__host__ __device__ inline int tc_resid_bytes(int resid_tma, int half) { return resid_tma ? 2 * (half / 64) * 16384 : 0; }

// One 128-row tile per CTA, split over two consumer warpgroups (rows 0-63 / 64-127), each holding its 64 x BN accumulator in
// registers.  BN (accumulator columns per CTA) is a template parameter so that each product of a k-step is ONE wgmma
// m64nBNk16: the A tile is read from shared memory once per product instead of once per 64 columns, and no run-time
// width switch sits between the MMAs.
template <int TC_BK, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_ln_tc_kernel(const __grid_constant__ CUtensorMap mapA_hi, const __grid_constant__ CUtensorMap mapA_lo,
                  const __grid_constant__ CUtensorMap mapW_hi, const __grid_constant__ CUtensorMap mapW_lo,
                  const __grid_constant__ CUtensorMap mapX_hi, const __grid_constant__ CUtensorMap mapX_lo,
                  const __grid_constant__ CUtensorMap mapO_hi, const __grid_constant__ CUtensorMap mapO_lo,
                  const TcArgs a) {
    extern __shared__ uint8_t smem_raw[];
    // aligned by an offset from smem_raw (not through an integer), so that the compiler keeps shared-memory loads
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    pdl_launch_dependents();          // PDL: let the next kernel's CTAs be scheduled behind this one

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;                                 // 0: producer warpgroup, 1 / 2: consumers of rows 0-63 / 64-127
    if (threadIdx.x == 0) dbg_time(a.dbg, 8);                        // t0: kernel entry
    const int rank = (int)cluster_ctarank();                         // channel slice of this CTA
    const int ncta = (int)cluster_nctarank();
    const int nslices = ncta;
    constexpr int MAXC = tc_max_cluster(BN);                         // cluster size bound: the statistics merge's unroll
    constexpr int bn = BN;                                           // accumulator columns per CTA
    const int half = a.half;                                         // columns per LN half (mode 0: bn)
    constexpr int HALF = BN / 2, NG = BN / 8, HG = BN / 16;          // modes 1, 2: columns of one LN half; 8-column groups
    constexpr int TC_A_PLANE = TC_BM * TC_BK * 2;                    // bytes of one activation plane tile
    constexpr int SW = TC_BK * 2;                                    // swizzle span = row bytes (128 or 64)
    constexpr int b_plane = bn * SW;                                 // bytes of one weight plane tile
    constexpr int A_BYTES = 2 * TC_A_PLANE;                          // hi+lo planes
    constexpr int stage_bytes = A_BYTES + 2 * b_plane;
    const int stages = a.stages;
    const int nkb = a.ntaps * a.kb_per_tap;

    uint8_t* rs = smem + tc_ring_bytes(stages, stage_bytes);      // residual / output staging tile
    uint8_t* aux = rs + tc_resid_bytes(a.resid_tma, half);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);              // [stages]
    uint64_t* empty_bar = full_bar + TC_MAX_STAGES;                      // [stages]
    uint64_t* resid_bar = empty_bar + TC_MAX_STAGES;
    float* s_bias = reinterpret_cast<float*>(aux + 256);
    float* s_gam = s_bias + 512;
    float* s_bet = s_gam + 512;
    float4* s_part = reinterpret_cast<float4*>(s_bet + 512);            // [128 rows]: this CTA's partial (sum, M2) x 2 halves, read by its peers

    pdl_wait();                       // upstream grid complete, its writes visible
    // ---- tile coordinates (a tile index past the end loads zeros and stores nothing) ----
    const int L = a.win.L;
    int t_end, t_lo;
    if (a.win.jptr) { t_end = __ldg(a.win.jptr); t_lo = max(0, t_end - a.win.R + 1); }
    else { t_end = L - 1; t_lo = 0; }
    int b0s, t0s;
    {
        const int tile = blockIdx.y;
        const int bg = tile / a.tiles_t, tt = tile - bg * a.tiles_t;
        b0s = (tile < a.ntiles) ? bg * a.TB : a.win.B;                  // batch coordinate out of range -> TMA zero fill
        t0s = a.win.jptr ? (t_end - a.tiles_t * a.TT + 1 + tt * a.TT) : tt * a.TT;
    }
    const bool mcast = a.mcast != 0 && ncta > 1;

    // ---- one-time setup ----
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&mapA_hi); prefetch_tmap(&mapA_lo); prefetch_tmap(&mapW_hi); prefetch_tmap(&mapW_lo);
        // each consumer warpgroup releases a stage once; with the multicast A tile a stage may only be refilled once EVERY
        // CTA of the cluster has drained it, so the consumers arrive on all CTAs' empty barriers
        for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], mcast ? 2u * (uint32_t)ncta : 2u); }
        mbar_init(resid_bar, 1);
        fence_mbar_init();
    }
    // epilogue vectors, indexed by accumulator column
    for (int c = threadIdx.x; c < bn; c += TC_THREADS) {
        float bi = 0.f, g = 0.f, be = 0.f;
        if (a.mode == 0) {
            int col = rank * bn + c;
            if (col < a.C) { bi = a.bias[col]; g = a.g1[col]; be = a.b1[col]; }
        } else {
            int second = c >= half;
            int col = rank * half + (second ? c - half : c);
            bi = (a.mode == 1 && second) ? a.bias[a.C + col] : a.bias[col];
            g = second ? a.g2[col] : a.g1[col];
            be = second ? a.b2[col] : a.b1[col];
        }
        s_bias[c] = bi; s_gam[c] = g; s_bet[c] = be;
    }
    __syncthreads();
    if (threadIdx.x == 0) { dbg_mark(a.dbg, 0, 1); dbg_mark(a.dbg, 2, nkb); dbg_time(a.dbg, 9); }   // t1: setup done
    if (ncta > 1) { cluster_arrive(); cluster_wait(); }   // phase 1: every CTA is running, its barriers initialised
    const uint16_t cta_mask = (uint16_t)((1u << ncta) - 1u);
    const int slice_rows = TC_BM / ncta;

    if (wg == 0) {
        // =========================== TMA producer ===========================
        // its registers go to the consumers, whose epilogue holds the whole fragment: 128 x 40 + 256 x 232 = 64,512
        // registers, what __launch_bounds__(384, 1) gives the CTA
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % stages;
                const uint32_t ph = (uint32_t)(kb / stages) & 1u;
                mbar_wait(&empty_bar[s], ph ^ 1u);
                mbar_expect_tx(&full_bar[s], (uint32_t)stage_bytes);
                uint8_t* st = smem + (size_t)s * stage_bytes;
                const int tap = kb / a.kb_per_tap, kc = kb - tap * a.kb_per_tap;
                const int tcoord = t0s + a.shifts[tap];
                if (mcast) {
                    // this CTA fetches rows [rank*slice, +slice) of the tile for the whole cluster
                    const int off = rank * slice_rows * SW;
                    tma_load_3d_mc(&mapA_hi, &full_bar[s], st + off, kc * TC_BK, tcoord + rank * slice_rows, b0s, cta_mask);
                    tma_load_3d_mc(&mapA_lo, &full_bar[s], st + TC_A_PLANE + off, kc * TC_BK, tcoord + rank * slice_rows, b0s, cta_mask);
                } else {
                    tma_load_3d(&mapA_hi, &full_bar[s], st, kc * TC_BK, tcoord, b0s);
                    tma_load_3d(&mapA_lo, &full_bar[s], st + TC_A_PLANE, kc * TC_BK, tcoord, b0s);
                }
                tma_load_2d(&mapW_hi, &full_bar[s], st + A_BYTES, kb * TC_BK, rank * bn);
                tma_load_2d(&mapW_lo, &full_bar[s], st + A_BYTES + b_plane, kb * TC_BK, rank * bn);
            }
            dbg_mark(a.dbg, 3, nkb);
            if (a.resid_tma) {
                // highway residual = this CTA's 'half' channels of the same rows, into its own staging tile: it arrives
                // while the k-blocks are still being multiplied
                const int nbox = half / 64;
                mbar_expect_tx(resid_bar, (uint32_t)(2 * nbox * 16384));
                for (int i = 0; i < nbox; ++i) {
                    tma_load_3d(&mapX_hi, resid_bar, rs + i * 16384, rank * half + i * 64, t0s, b0s);
                    tma_load_3d(&mapX_lo, resid_bar, rs + (nbox + i) * 16384, rank * half + i * 64, t0s, b0s);
                }
            }
        }
        __syncwarp();
    } else {
        // =========================== wgmma consumers ===========================
        setmaxnreg_inc<232>();
        const int mh = wg - 1;                                           // row half of the tile
        float acc[BN / 2];                                               // m64nBN fragment (tc_ptx.cuh)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        // stage s is drained: let the producer(s) refill it.  With the multicast A tile every CTA of the cluster waits for
        // this release, and thread p of the warpgroup signals CTA p, so the cluster-scope arrives go out side by side
        // instead of one after another on a single thread
        auto release = [&](int s) {
            const int t = threadIdx.x & 127;
            if (mcast) { if (t < ncta) mbar_arrive_cluster(&empty_bar[s], (uint32_t)t); }
            else if (t == 0) mbar_arrive(&empty_bar[s]);
        };
        for (int kb = 0; kb < nkb; ++kb) {
            const int s = kb % stages;
            mbar_wait(&full_bar[s], (uint32_t)(kb / stages) & 1u);
            const uint32_t st = smem_u32(smem + (size_t)s * stage_bytes);
            const uint64_t dA_hi = gmma_desc_kmajor<SW>(st + mh * 64 * SW), dA_lo = gmma_desc_kmajor<SW>(st + TC_A_PLANE + mh * 64 * SW);
            const uint64_t dB_hi = gmma_desc_kmajor<SW>(st + A_BYTES), dB_lo = gmma_desc_kmajor<SW>(st + A_BYTES + b_plane);
            wg_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 16; ++k) {
                const uint64_t adv = (uint64_t)(k * 32 >> 4);            // 16 fp16 = 32 B inside the swizzle atom
                wgmma_full<BN>(acc, dA_hi + adv, dB_hi + adv, (kb | k) != 0);
                wgmma_full<BN>(acc, dA_hi + adv, dB_lo + adv, 1u);
                wgmma_full<BN>(acc, dA_lo + adv, dB_hi + adv, 1u);
            }
            wg_commit();
            // keep this k-block's MMAs in flight; the previous one is finished once at most one group is pending
            wg_wait<1>();
            if (kb > 0) release((kb - 1) % stages);
        }
        wg_wait<0>();                                                    // the last k-block (its stage is never refilled)
        wg_fence_regs(acc);
        if (threadIdx.x == 128) { dbg_mark(a.dbg, 4, nkb); dbg_mark(a.dbg, 5, 1); dbg_time(a.dbg, 10); }   // t2: main loop over

        // =========================== epilogue on the fragment: both warpgroups, 64 rows each ===========================
        const int j = lane & 3;
        const int rt = mh * 64 + (warp & 3) * 16 + (lane >> 2);          // tile rows rt (h = 0) and rt + 8 (h = 1)
        int bb[2], tt[2];
        bool ok[2], live[2];
        float inv_s[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = rt + 8 * h, bi = r / a.TT;
            const int b = b0s + bi, t = t0s + r - bi * a.TT;
            bb[h] = b; tt[h] = t;
            ok[h] = (b < a.win.B) && (t >= t_lo) && (t <= t_end) && (t < L);
            // ragged launch: a row at or past its utterance's length (in this block's input rows) is stored as zeros, so
            // that the next block's taps read there what TMA's zero fill gives a launch over the utterance alone
            live[h] = !(a.lengths && b < a.win.B) || t < (min(max(__ldg(a.lengths + b), 0), L >> a.len_shift) << a.len_shift);
            // a row reads input rows of its own utterance only, so one input scale per row; both scales are powers of two
            inv_s[h] = a.inv_scale * ((a.in_inv && b < a.win.B) ? __ldg(a.in_inv + b) : 1.f);
        }
#pragma unroll
        for (int q = 0; q < NG; ++q) {
            const float2 bi2 = *reinterpret_cast<const float2*>(s_bias + 8 * q + 2 * j);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                acc[4 * q + 2 * h] = fmaf(acc[4 * q + 2 * h], inv_s[h], bi2.x);
                acc[4 * q + 2 * h + 1] = fmaf(acc[4 * q + 2 * h + 1], inv_s[h], bi2.y);
            }
        }
        const int n1 = (a.mode == 0) ? min(max(a.C - rank * bn, 0), bn) : HALF;

        float s1[2], q1[2], s2[2] = {0.f, 0.f}, q2[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (a.mode == 0) row_stats<0, NG>(acc, h, j, n1, s1[h], q1[h]);
            else { row_stats<0, HG>(acc, h, j, HALF, s1[h], q1[h]); row_stats<HG, HG>(acc, h, j, HALF, s2[h], q2[h]); }
        }
        // combine over the cluster
        float mean1[2], rstd1[2], mean2[2] = {0.f, 0.f}, rstd2[2] = {0.f, 0.f};
        if (ncta > 1) {
            // each CTA publishes its partials in its OWN shared memory; after the cluster barrier every CTA reads
            // the slices' partials through distributed shared memory
            if (j == 0) {
                s_part[rt] = make_float4(s1[0], q1[0], s2[0], q2[0]);
                s_part[rt + 8] = make_float4(s1[1], q1[1], s2[1], q2[1]);
            }
            if (threadIdx.x == 128) { dbg_mark(a.dbg, 6, 1); dbg_time(a.dbg, 11); }   // t3: statistics done, partials published
            cluster_arrive();                                              // phase 2: partials published
            cluster_wait();
            if (threadIdx.x == 128) { dbg_mark(a.dbg, 7, 1); dbg_time(a.dbg, 12); }   // t4: cluster barrier passed
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t my_slot = smem_u32(&s_part[rt + 8 * h]);
                float4 pv[MAXC];
#pragma unroll
                for (int p = 0; p < MAXC; ++p) pv[p] = (p < nslices) ? ld_cluster_f4(mapa(my_slot, (uint32_t)p)) : make_float4(0.f, 0.f, 0.f, 0.f);
                float S1 = 0.f, S2 = 0.f;
#pragma unroll
                for (int p = 0; p < MAXC; ++p) if (p < nslices) { S1 += pv[p].x; S2 += pv[p].z; }
                mean1[h] = S1 / (float)a.C; mean2[h] = S2 / (float)a.C;
                float M1 = 0.f, M2 = 0.f;
#pragma unroll
                for (int p = 0; p < MAXC; ++p) {
                    if (p >= nslices) continue;
                    const float4 v = pv[p];
                    const int np = (a.mode == 0) ? min(max(a.C - p * bn, 0), bn) : HALF;
                    if (np > 0) { float d = v.x / (float)np - mean1[h]; M1 += v.y + (float)np * d * d; }
                    if (a.mode != 0) { float d = v.z / (float)HALF - mean2[h]; M2 += v.w + (float)HALF * d * d; }
                }
                rstd1[h] = 1.0f / sqrtf(M1 / (float)a.C + 1e-12f);
                rstd2[h] = 1.0f / sqrtf(M2 / (float)a.C + 1e-12f);
            }
        } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                mean1[h] = n1 > 0 ? s1[h] / (float)max(n1, 1) : 0.f; rstd1[h] = 1.0f / sqrtf(q1[h] / (float)a.C + 1e-12f);
                mean2[h] = s2[h] / (float)HALF; rstd2[h] = 1.0f / sqrtf(q2[h] / (float)a.C + 1e-12f);
            }
        }

        // normalise, activate, mix, store
        if (a.mode == 0) {
#pragma unroll
            for (int q = 0; q < NG; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * q + 2 * j + e;
                        float z = (acc[4 * q + 2 * h + e] - mean1[h]) * rstd1[h] * s_gam[c] + s_bet[c];
                        if (a.act == 1) z = fmaxf(z, 0.f);
                        acc[4 * q + 2 * h + e] = (c < n1 && live[h]) ? z : 0.f;
                    }
            const int col0 = rank * bn;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const size_t row = (size_t)bb[h] * L + tt[h];
                if (a.out.hi) store_planes_frag<0, NG>(a.out, row, col0, acc, h, j, ok[h]);
                if (ok[h] && a.out_f32) store_f32_frag<0, NG>(a.out_f32 + row * a.ld_f32, col0, n1, acc, h, j);
            }
            if (a.sig_f32 || a.sig.hi) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int q = 0; q < NG; ++q)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = 8 * q + 2 * j + e;
                            acc[4 * q + 2 * h + e] = (c < n1 && live[h]) ? sigmoid_acc(acc[4 * q + 2 * h + e]) : 0.f;
                        }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const size_t row = (size_t)bb[h] * L + tt[h];
                    if (a.sig.hi) store_planes_frag<0, NG>(a.sig, row, col0, acc, h, j, ok[h]);
                    if (ok[h] && a.sig_f32) store_f32_frag<0, NG>(a.sig_f32 + row * a.ld_sig, col0, n1, acc, h, j);
                }
            }
        } else if (a.mode == 1) {
            // residual / output staging tile: [plane][box of 64 ch][128 rows][128 B], 128B swizzle; the pair of columns a
            // thread holds in a row is 4 bytes of one 16-byte chunk, and the 8 rows of a warp's access hit 8 distinct chunks
            const int nbox = HALF / 64;
            if (a.resid_tma) mbar_wait(resid_bar, 0);
#pragma unroll
            for (int q = 0; q < HG; ++q) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rt + 8 * h;
                    const size_t row = (size_t)bb[h] * L + tt[h];
                    const int c = 8 * q + 2 * j;
                    uint8_t* sh = rs + (q >> 3) * 16384 + r * 128 + ((((q & 7) ^ (r & 7)) << 4) | (4 * j));
                    uint8_t* sl = sh + nbox * 16384;
                    __half2 xh = __float2half2_rn(0.f), xl = xh;
                    if (a.resid_tma) {
                        xh = *reinterpret_cast<const __half2*>(sh);
                        xl = *reinterpret_cast<const __half2*>(sl);
                    } else if (ok[h]) {
                        xh = __ldg(reinterpret_cast<const __half2*>(a.X.hi + row * a.X.ld + rank * HALF + c));
                        xl = __ldg(reinterpret_cast<const __half2*>(a.X.lo + row * a.X.ld + rank * HALF + c));
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float z1 = (acc[4 * q + 2 * h + e] - mean1[h]) * rstd1[h] * s_gam[c + e] + s_bet[c + e];
                        const float z2 = (acc[4 * (q + HG) + 2 * h + e] - mean2[h]) * rstd2[h] * s_gam[HALF + c + e] + s_bet[HALF + c + e];
                        const float h1 = sigmoid_acc(z1);
                        const float x = e ? join_f16(__high2half(xh), __high2half(xl)) : join_f16(__low2half(xh), __low2half(xl));
                        acc[4 * q + 2 * h + e] = live[h] ? h1 * z2 + (1.0f - h1) * x : 0.f;
                    }
                    if (a.out_tma) {
                        // stage the output planes in place of the residual just consumed (same swizzled slots)
                        __half2 oh, ol;
                        split_f16x2(make_float2(acc[4 * q + 2 * h], acc[4 * q + 2 * h + 1]), oh, ol);
                        *reinterpret_cast<__half2*>(sh) = oh;
                        *reinterpret_cast<__half2*>(sl) = ol;
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const size_t row = (size_t)bb[h] * L + tt[h];
                if (!a.out_tma && a.out.hi) store_planes_frag<0, HG>(a.out, row, rank * HALF, acc, h, j, ok[h]);
                if (ok[h] && a.out_f32) store_f32_frag<0, HG>(a.out_f32 + row * a.ld_f32, rank * HALF, HALF, acc, h, j);
            }
            if (a.out_tma) {
                // whole tile staged: one thread hands it to the TMA engine (rows past the end are clipped)
                fence_proxy_async_smem();
                named_sync(1, 256);                                          // both consumer warpgroups
                if (threadIdx.x == 128) {
                    for (int i = 0; i < nbox; ++i) {
                        tma_store_3d(&mapO_hi, rs + i * 16384, rank * HALF + i * 64, t0s, b0s);
                        tma_store_3d(&mapO_lo, rs + (nbox + i) * 16384, rank * HALF + i * 64, t0s, b0s);
                    }
                    tma_store_commit_and_wait();
                }
            }
        } else {
            // transposed conv: first half -> output row 2t, second half -> row 2t+1 (modules.py:232-241)
#pragma unroll
            for (int q = 0; q < NG; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * q + 2 * j + e;
                        const float mean = q < HG ? mean1[h] : mean2[h], rstd = q < HG ? rstd1[h] : rstd2[h];
                        acc[4 * q + 2 * h + e] = live[h] ? (acc[4 * q + 2 * h + e] - mean) * rstd * s_gam[c] + s_bet[c] : 0.f;
                    }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const size_t row_e = (size_t)bb[h] * (2 * L) + 2 * (size_t)tt[h];
                if (a.out.hi) {
                    store_planes_frag<0, HG>(a.out, row_e, rank * HALF, acc, h, j, ok[h]);
                    store_planes_frag<HG, HG>(a.out, row_e + 1, rank * HALF, acc, h, j, ok[h]);
                }
                if (ok[h] && a.out_f32) {
                    store_f32_frag<0, HG>(a.out_f32 + row_e * a.ld_f32, rank * HALF, HALF, acc, h, j);
                    store_f32_frag<HG, HG>(a.out_f32 + (row_e + 1) * a.ld_f32, rank * HALF, HALF, acc, h, j);
                }
            }
        }
        if (threadIdx.x == 128) dbg_time(a.dbg, 13);                      // t5: stores issued
    }

    // ---- teardown: the producer warpgroup matches the consumers' cluster barrier phase ----
    if (ncta > 1) {
        if (wg == 0) { cluster_arrive(); cluster_wait(); }
        cluster_arrive();                     // last phase: nobody reads my shared memory any more
        cluster_wait();
    }
    if (threadIdx.x == 0) dbg_time(a.dbg, 14);                            // t6: teardown barrier passed
}

// ------------------------------------------------------------------------------------------
// plane conversion kernels (boundaries of the tensor-core path)
// ------------------------------------------------------------------------------------------
__global__ void f32_to_planes_kernel(const float* __restrict__ x, int ldx, Planes p, long long rows, int C) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = rows * C;
    if (i >= total) return;
    long long r = i / C; int c = (int)(i - r * C);
    split_f16(x[r * ldx + c], p.hi[r * p.ld + c], p.lo[r * p.ld + c]);
}
__global__ void planes_to_f32_kernel(Planes p, float* __restrict__ y, int ldy, long long rows, int C) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = rows * C;
    if (i >= total) return;
    long long r = i / C; int c = (int)(i - r * C);
    y[r * ldy + c] = join_f16(p.hi[r * p.ld + c], p.lo[r * p.ld + c]);
}
// One CTA per utterance: abs-max of its L x C inputs -> s = utterance_scale(max), then the planes of s x.  With lengths,
// only the utterance's first lengths[b] rows (clamped to [0, L]) are read; its rows past them become zero planes, which is
// what the TMA zero fill gives a call over those rows alone.
constexpr int PLANES_SCALED_THREADS = 512;
__global__ void __launch_bounds__(PLANES_SCALED_THREADS)
f32_to_planes_scaled_kernel(const float* __restrict__ x, int ldx, Planes p, int L, int C, float* __restrict__ in_inv,
                            const int* __restrict__ lengths) {
    __shared__ float s_red[PLANES_SCALED_THREADS / 32];
    __shared__ float s_scale;
    const int b = blockIdx.x, n = L * C;
    const int nlive = lengths ? min(max(__ldg(lengths + b), 0), L) * C : n;
    const float* xb = x + (size_t)b * L * ldx;
    float m = 0.f;
    for (int i = threadIdx.x; i < nlive; i += blockDim.x) {
        const int r = i / C, c = i - r * C;
        m = fmaxf(m, fabsf(xb[(size_t)r * ldx + c]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, s_red[w]);
        const float sc = utterance_scale(m);
        s_scale = sc;
        in_inv[b] = 1.f / sc;
    }
    __syncthreads();
    const float sc = s_scale;
    const size_t row0 = (size_t)b * L;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int r = i / C, c = i - r * C;
        split_f16(i < nlive ? xb[(size_t)r * ldx + c] * sc : 0.f, p.hi[(row0 + r) * p.ld + c], p.lo[(row0 + r) * p.ld + c]);
    }
}
void launch_f32_to_planes(const float* x, int ldx, Planes p, long long rows, int C, cudaStream_t s) {
    long long n = rows * C;
    if (n > 0) f32_to_planes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, ldx, p, rows, C);
}
void launch_f32_to_planes_scaled(const float* x, int ldx, Planes p, int B, int L, int C, float* in_inv, cudaStream_t s,
                                 const int* lengths) {
    if (B > 0 && (long long)L * C > 0x7fffffffLL) throw std::runtime_error("f32_to_planes_scaled: L x C exceeds 2^31");
    if (B > 0) f32_to_planes_scaled_kernel<<<(unsigned)B, PLANES_SCALED_THREADS, 0, s>>>(x, ldx, p, L, C, in_inv, lengths);
}
// grid (x: row blocks, y: windows); the product and split are f32_to_planes_scaled_kernel's, with the scale fixed
__global__ void mel_windows_to_planes_kernel(const float* __restrict__ Y, int T, int C, const int* __restrict__ win, int W,
                                             int L, Planes p, float* __restrict__ in_inv) {
    const int w = blockIdx.y;
    const int n = __ldg(win + w), utt = __ldg(win + W + w), row0 = __ldg(win + 2 * W + w);
    if (blockIdx.x == 0 && threadIdx.x == 0) in_inv[w] = 1.f / SSRN_WINDOW_SCALE;
    const float* yb = Y + ((size_t)utt * T + row0) * C;
    const size_t prow = (size_t)w * L;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L * C; i += gridDim.x * blockDim.x) {
        const int r = i / C, c = i - r * C;
        split_f16(r < n ? yb[(size_t)r * C + c] * SSRN_WINDOW_SCALE : 0.f, p.hi[(prow + r) * p.ld + c], p.lo[(prow + r) * p.ld + c]);
    }
}
void launch_mel_windows_to_planes(const float* Y, int T, int C, const int* win, int W, int L, Planes p, float* in_inv,
                                  cudaStream_t s) {
    if (W <= 0 || L <= 0) return;
    const int blocks = std::min(64, (L * C + 255) / 256);
    mel_windows_to_planes_kernel<<<dim3((unsigned)blocks, (unsigned)W), 256, 0, s>>>(Y, T, C, win, W, L, p, in_inv);
}
void launch_planes_to_f32(Planes p, float* y, int ldy, long long rows, int C, cudaStream_t s) {
    long long n = rows * C;
    if (n > 0) planes_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, y, ldy, rows, C);
}

// ------------------------------------------------------------------------------------------
// host side: tensor maps and the cluster launch
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
            throw std::runtime_error("cuTensorMapEncodeTiled is not available from the driver");
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

void tc_make_act_map(CUtensorMap* m, const __half* base, int C, int ld, int L, int B, int TT, int TB, int bk) {
    cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)L, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)L * ld * 2};
    cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)TT, (cuuint32_t)TB};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<__half*>(base), dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(activation) failed: " + std::to_string((int)r));
}

// generic rank-3 fp16 map: dims {d0, d1, d2} (d0 contiguous), byte strides of d1 / d2, box {b0, b1, 1}; the swizzle follows the
// box's inner extent (64 elements -> 128 bytes, 32 -> 64 bytes), out-of-range coordinates (negative too) read zeros
void tc_make_map3(CUtensorMap* m, const __half* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                  uint64_t stride2_bytes, uint32_t b0, uint32_t b1) {
    cuuint64_t dims[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
    cuuint64_t strides[2] = {(cuuint64_t)stride1_bytes, (cuuint64_t)stride2_bytes};
    cuuint32_t box[3] = {(cuuint32_t)b0, (cuuint32_t)b1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (b0 != 64 && b0 != 32) throw std::runtime_error("tc_make_map3: the inner box extent must be 32 or 64 halfs");
    CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<__half*>(base), dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, b0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(map3) failed: " + std::to_string((int)r));
}

void tc_make_w_map(CUtensorMap* m, const __half* base, int Ktot, int Nrows, int bn, int bk) {
    cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)Nrows};
    cuuint64_t strides[1] = {(cuuint64_t)Ktot * 2};
    cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)bn};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r));
}

int tc_bk() {
    // 32-wide slabs (64-byte swizzle): beside the highway residual tile (64 KB) of a 256-column block there is room for three
    // 48 KB stages, where 64-wide stages (96 KB) would fit only one
    return 32;
}

static size_t conv_ln_smem(int stages, int bn, int half, int resid_tma, int bk) {
    const int stage = 2 * TC_BM * bk * 2 + 2 * bn * bk * 2;
    return (size_t)tc_ring_bytes(stages, stage) + tc_resid_bytes(resid_tma, half) + TC_AUX_BYTES + 1024;
}

int tc_stages_for(int bn, int bk, int resid_tma, int half) {      // bn = accumulator columns per CTA
    int s = TC_MAX_STAGES;
    while (s > 2 && conv_ln_smem(s, bn, half, resid_tma, bk) > (size_t)TC_MAX_SMEM) --s;
    return s;
}

// the kernel instantiation for (bk, bn): the accumulator widths of the networks' blocks -- 64 (Text2Mel's 256-channel
// blocks), 80 (the mel output), 144 (the F = 1025 blocks over 8 CTAs, F = 2049 over 16), 256 (the 512- and 1024-channel
// blocks)
typedef void (*ConvLnKernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                             const CUtensorMap, const CUtensorMap, const CUtensorMap, const TcArgs);
template <int BK>
static ConvLnKernel conv_ln_kernel_bn(int bn) {
    switch (bn) {
        case 64: return conv_ln_tc_kernel<BK, 64>;
        case 80: return conv_ln_tc_kernel<BK, 80>;
        case 144: return conv_ln_tc_kernel<BK, 144>;
        case 256: return conv_ln_tc_kernel<BK, 256>;
        default: throw std::runtime_error("conv_ln_tc: no kernel for " + std::to_string(bn) + " accumulator columns per CTA "
                                          "(64, 80, 144, 256)");
    }
}

// The instantiation for (bk, bn) with its attributes raised on the current device: the shared-memory limit, and for the
// 144-column one clusters of 16 CTAs
static ConvLnKernel conv_ln_kernel_ready(int bk, int bn) {
    const ConvLnKernel kern = bk == 64 ? conv_ln_kernel_bn<64>(bn) : conv_ln_kernel_bn<32>(bn);
    // the attributes are per device and per instantiation: cache them per device, not per process (a second Engine on
    // another GPU of the same process must raise its own limits)
    static bool attr_set_dev[64][8] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    const int inst = (bk == 64 ? 4 : 0) + (bn == 64 ? 0 : bn == 80 ? 1 : bn == 144 ? 2 : 3);
    bool& attr_set = attr_set_dev[dev & 63][inst];
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_MAX_SMEM);
        if (e == cudaSuccess && tc_max_cluster(bn) > 8) e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        if (e != cudaSuccess) throw std::runtime_error(std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e));
        attr_set = true;
    }
    return kern;
}

int conv_ln_tc_max_clusters(int ncta, int bn, int bk) {
    const ConvLnKernel kern = conv_ln_kernel_ready(bk, bn);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ncta, 1, 1);
    cfg.blockDim = dim3(TC_THREADS, 1, 1);
    cfg.dynamicSmemBytes = conv_ln_smem(tc_stages_for(bn, bk, 0, bn), bn, bn, 0, bk);
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)ncta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

void launch_conv_ln_tc(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi,
                       const CUtensorMap& w_lo, const CUtensorMap* io, const TcArgs& a, int ncta, int ctas_y, int bk,
                       cudaStream_t s) {
    if (ncta > tc_max_cluster(a.bn))
        throw std::runtime_error("conv_ln_tc: a cluster of " + std::to_string(ncta) + " CTAs at " + std::to_string(a.bn) +
                                 " columns (16 at 144 columns, else 8 at most)");
    if (a.mode != 0 && 2 * a.half != a.bn) throw std::runtime_error("conv_ln_tc: hc and transposed blocks hold two halves of bn / 2 columns");
    const ConvLnKernel kern = conv_ln_kernel_ready(bk, a.bn);
    const size_t smem = conv_ln_smem(a.stages, a.bn, a.half, a.resid_tma, bk);
    if (smem > (size_t)TC_MAX_SMEM) throw std::runtime_error("conv_ln_tc: shared memory budget exceeded");
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ncta, (unsigned)ctas_y, 1);
    cfg.blockDim = dim3(TC_THREADS, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)ncta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 2 : 1;
    if (a.resid_tma && !io) throw std::runtime_error("conv_ln_tc: residual TMA needs the X / out tensor maps");
    const CUtensorMap& x_hi = io ? io[0] : a_hi;      // unused placeholders when resid_tma == 0
    const CUtensorMap& x_lo = io ? io[1] : a_lo;
    const CUtensorMap& o_hi = io ? io[2] : a_hi;
    const CUtensorMap& o_lo = io ? io[3] : a_lo;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, a_hi, a_lo, w_hi, w_lo, x_hi, x_lo, o_hi, o_lo, a);
    if (e != cudaSuccess) throw std::runtime_error(std::string("conv_ln_tc launch: ") + cudaGetErrorString(e));
}

}  // namespace dctts
