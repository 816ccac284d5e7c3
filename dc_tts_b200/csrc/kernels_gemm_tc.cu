// kernels_gemm_tc.cu -- the three conv-GEMMs of the training step (reference train.py:122-132 runs them inside
// tf.train.AdamOptimizer.compute_gradients: forward conv1d, its data gradient and its weight gradient) on the
// 5th-generation tensor cores, with fp32 tensors on both sides.
//
//   forward / data gradient (mode 0):  Y[b,t,n] (+)= bias[n] + sum_tap sum_k X[b, t+shift_tap, k] W_tap[k][n]
//   weight gradient        (mode 1):  dW[tap][k][n] += sum_b sum_t X[b, t+shift_tap, k] dY[b,t,n]
//
// fp32 operands cannot feed the tensor cores directly, and bf16 / single fp16 operands miss the gradient-parity budget, so every
// operand is first written as split-fp16 planes with a per-tensor scale (numerics.cuh: the format and slot_scale).  The planes
// are laid out so that BOTH operands of all three GEMMs are K-major tiles that TMA delivers in the 64-byte swizzle, the
// reduction index being contiguous:
//   mode 0: A = activation planes (B, L, C) box {32 ch, 128 t, 1 b}: the conv tap is the box's time coordinate and TMA's
//           zero fill is the zero padding;  B = weight planes [n][tap * Kp + k].
//   mode 1: A = TRANSPOSED activation planes (tap, B, C, L) box {32 t, 128 k, 1 b} (one pre-shifted copy per tap), B = transposed
//           gradient planes (B, N, L) box {32 t, bn n, 1 b}; the reduction runs over (b, t-block), split over CTAs, and the
//           partial tiles are added to dW with vector reductions (red.global.add.v4.f32) -- or, in the ordered mode
//           (kernels_ordered.cu), stored to part[split][tap][K][ldp] and added up in split order by the ordered reduction.
// One 128 x bn accumulator tile per CTA (bn <= 256), 32-wide slabs, up to four pipeline stages.  Warp 0 = TMA producer,
// warpgroups 1 and 2 = wgmma consumers of rows 0-63 / 64-127 (fp32 register accumulators), which then write the tile to
// shared memory (over the drained ring) and store it one row per thread, each warpgroup half of the columns.
#include "kernels.cuh"
#include "kernels_tc.cuh"
#include "numerics.cuh"
#include "tc_ptx.cuh"

#include <algorithm>
#include <stdexcept>
#include <string>

namespace dctts {
using namespace ptx;

namespace {

constexpr int G_BM = 128, G_BK = 32, G_THREADS = 384, G_MAX_STAGES = 4;
constexpr int G_SW = G_BK * 2;                         // bytes per tile row = swizzle span (64)
constexpr int G_APLANE = G_BM * G_SW;                  // one plane of the A tile (8 KB)
constexpr int G_AUX = 256;

struct GemmTcArgs {
    int mode;                 // 0: rows x channels conv GEMM, 1: weight gradient
    int bn;                   // accumulator columns per CTA (multiple of 16, <= 256)
    int stages;
    // mode 0
    int L, Lout, tiles_t, ntaps, kb_per_tap, Kp2, N;
    int shifts[3];
    float* Y; int ldy; const float* bias; int accumulate;
    // mode 1
    int tblocks, nb_per_split, B, ksplit, K;
    float* dW; int ldw; long long tap_stride;
    const unsigned* slot_a; const unsigned* slot_b;
    float* part; int ldp;     // mode 1, ordered: the split tiles go to part (null: added to dW)
    int probe;                // measurement only: 1 = the operands are fetched but no MMA is issued and nothing is stored
};

__host__ __device__ inline int g_acc_ld(int bn) { return bn + 4; }
// ring of `stages` stages, reused after the main loop for the 128 x (bn + 4) fp32 accumulator tile
__host__ __device__ inline int g_ring_bytes(int stages, int bn) {
    const int ring = stages * (2 * G_APLANE + 2 * bn * G_SW) + 64 * G_SW;      // a 64-column wgmma past bn reads <= 48 rows more
    const int acc = G_BM * g_acc_ld(bn) * 4;
    return ((ring > acc ? ring : acc) + 1023) & ~1023;
}

// PART: mode 1 in the ordered mode, the split tiles stored to a.part (a separate instantiation, so that the default
// kernel's code is not touched by it)
template <bool PART>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA_hi, const __grid_constant__ CUtensorMap mapA_lo,
               const __grid_constant__ CUtensorMap mapB_hi, const __grid_constant__ CUtensorMap mapB_lo, const GemmTcArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int bn = a.bn, b_plane = bn * G_SW, stage_bytes = 2 * G_APLANE + 2 * b_plane, stages = a.stages;
    const int acc_ld = g_acc_ld(bn);
    float* s_acc = reinterpret_cast<float*>(smem);
    uint8_t* aux = smem + g_ring_bytes(stages, bn);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty_bar = full_bar + G_MAX_STAGES;

    // ---- tile coordinates and the reduction schedule ----
    const int n0 = blockIdx.x * bn;
    int b0 = 0, t0 = 0, tap = 0, nkb;
    if (a.mode == 0) {
        b0 = blockIdx.y / a.tiles_t; t0 = (blockIdx.y - b0 * a.tiles_t) * G_BM;
        nkb = a.ntaps * a.kb_per_tap;
    } else {
        tap = blockIdx.z / a.ksplit;
        b0 = (blockIdx.z - tap * a.ksplit) * a.nb_per_split;
        nkb = min(a.nb_per_split, a.B - b0) * a.tblocks;
    }
    if (nkb <= 0) return;                                           // uniform: an empty split has nothing to add
    const int m0 = blockIdx.y * G_BM;                               // mode 1: first input channel of the tile

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&mapA_hi); prefetch_tmap(&mapA_lo); prefetch_tmap(&mapB_hi); prefetch_tmap(&mapB_lo);
        for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }   // one release per consumer warpgroup
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 0) {
        // =========================== TMA producer ===========================
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % stages;
                mbar_wait(&empty_bar[s], (((uint32_t)(kb / stages)) & 1u) ^ 1u);
                mbar_expect_tx(&full_bar[s], (uint32_t)stage_bytes);
                uint8_t* st = smem + (size_t)s * stage_bytes;
                if (a.mode == 0) {
                    const int tp = kb / a.kb_per_tap, kc = kb - tp * a.kb_per_tap;
                    tma_load_3d(&mapA_hi, &full_bar[s], st, kc * G_BK, t0 + a.shifts[tp], b0);
                    tma_load_3d(&mapA_lo, &full_bar[s], st + G_APLANE, kc * G_BK, t0 + a.shifts[tp], b0);
                    tma_load_3d(&mapB_hi, &full_bar[s], st + 2 * G_APLANE, tp * a.Kp2 + kc * G_BK, n0, 0);
                    tma_load_3d(&mapB_lo, &full_bar[s], st + 2 * G_APLANE + b_plane, tp * a.Kp2 + kc * G_BK, n0, 0);
                } else {
                    const int bb = kb / a.tblocks, tb = kb - bb * a.tblocks;
                    tma_load_3d(&mapA_hi, &full_bar[s], st, tb * G_BK, m0, tap * a.B + b0 + bb);      // the tap's pre-shifted copy
                    tma_load_3d(&mapA_lo, &full_bar[s], st + G_APLANE, tb * G_BK, m0, tap * a.B + b0 + bb);
                    tma_load_3d(&mapB_hi, &full_bar[s], st + 2 * G_APLANE, tb * G_BK, n0, b0 + bb);
                    tma_load_3d(&mapB_lo, &full_bar[s], st + 2 * G_APLANE + b_plane, tb * G_BK, n0, b0 + bb);
                }
            }
        }
        __syncwarp();
        return;
    }
    if (wg == 0) return;                                            // warps 1-3: no role
    // =========================== wgmma consumers: rows 64 * (wg - 1) .. +64 ===========================
    const int mh = wg - 1;
    float acc[4][32];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % stages;
        mbar_wait(&full_bar[s], ((uint32_t)(kb / stages)) & 1u);
        if (!a.probe) {
            const uint32_t st = smem_u32(smem + (size_t)s * stage_bytes);
            const uint64_t dA_hi = gmma_desc_kmajor<G_SW>(st + mh * 64 * G_SW), dA_lo = gmma_desc_kmajor<G_SW>(st + G_APLANE + mh * 64 * G_SW);
            const uint64_t dB_hi = gmma_desc_kmajor<G_SW>(st + 2 * G_APLANE), dB_lo = gmma_desc_kmajor<G_SW>(st + 2 * G_APLANE + b_plane);
            wg_fence();
#pragma unroll
            for (int k = 0; k < G_BK / 16; ++k) {
                const uint64_t adv = (uint64_t)(k * 32 >> 4);          // 16 fp16 = 32 bytes inside the swizzle atom
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (j * 64 < bn) {
                        const uint64_t cb = (uint64_t)((j * 64 * G_SW) >> 4);
                        wgmma_split3(acc[j], min(64, bn - j * 64), dA_hi + adv, dA_lo + adv, dB_hi + cb + adv, dB_lo + cb + adv,
                                     (kb | k) != 0);
                    }
                }
            }
            wg_commit();
            wg_wait<0>();
#pragma unroll
            for (int j = 0; j < 4; ++j) wg_fence_regs(acc[j]);
        }
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[s]);     // stage drained (ingest probe: at once)
    }
    if (a.probe) return;
    named_sync(1, 256);                                             // both halves done reading the ring: it becomes the tile
    {
        const int r0 = mh * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i8 = 0; i8 < 8; ++i8) {
                const int col = j * 64 + i8 * 8 + 2 * (lane & 3);
                if (col < bn) {
                    *reinterpret_cast<float2*>(s_acc + (size_t)r0 * acc_ld + col) = make_float2(acc[j][i8 * 4], acc[j][i8 * 4 + 1]);
                    *reinterpret_cast<float2*>(s_acc + (size_t)(r0 + 8) * acc_ld + col) = make_float2(acc[j][i8 * 4 + 2], acc[j][i8 * 4 + 3]);
                }
            }
    }
    named_sync(1, 256);
    // =========================== epilogue: thread == accumulator row (both warpgroups, half the columns each) ===========================
    const int r = threadIdx.x & 127;
    const float* arow = s_acc + (size_t)r * acc_ld;
    const int c_beg = mh == 0 ? 0 : ((bn / 2 + 31) & ~31), c_end = mh == 0 ? ((bn / 2 + 31) & ~31) : bn;
    // both scales are powers of two up to 2^127: their product overflows for operands of max ~1e-16 (and would zero every
    // output), so the inverses are taken one at a time -- each is exact, and so is theirs down to 2^-149
    const float inv = (1.0f / slot_scale(a.slot_a)) * (1.0f / slot_scale(a.slot_b));
    if (a.mode == 0) {
        const int t = t0 + r;
        if (t < a.L) {
            float* yrow = a.Y + ((size_t)b0 * a.Lout + t) * a.ldy;
            for (int c = c_beg; c < c_end; c += 4) {
                const int n = n0 + c;
                const float4 v = *reinterpret_cast<const float4*>(arow + c);
                if (n + 3 < a.N) {
                    const float4 bq = __ldg(reinterpret_cast<const float4*>(a.bias + n));
                    float4 o = make_float4(fmaf(v.x, inv, bq.x), fmaf(v.y, inv, bq.y), fmaf(v.z, inv, bq.z), fmaf(v.w, inv, bq.w));
                    float4* p = reinterpret_cast<float4*>(yrow + n);
                    if (a.accumulate) { const float4 y = *p; o.x += y.x; o.y += y.y; o.z += y.z; o.w += y.w; }
                    *p = o;
                } else {
                    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (n + e < a.N) {
                            const float o = fmaf(vv[e], inv, __ldg(a.bias + n + e));
                            yrow[n + e] = a.accumulate ? yrow[n + e] + o : o;
                        }
                }
            }
        }
    } else {
        const int k = m0 + r;
        if (PART && k < a.K) {
            const int split = blockIdx.z - tap * a.ksplit, ntaps = gridDim.z / a.ksplit;
            float* prow = a.part + (((size_t)split * ntaps + tap) * a.K + k) * a.ldp;
            for (int c = c_beg; c < c_end; c += 4) {
                const int n = n0 + c;
                if (n < a.ldp) {
                    const float4 v = *reinterpret_cast<const float4*>(arow + c);
                    *reinterpret_cast<float4*>(prow + n) = make_float4(v.x * inv, v.y * inv, v.z * inv, v.w * inv);
                }
            }
        } else if (!PART && k < a.K) {
            float* wrow = a.dW + (size_t)tap * a.tap_stride + (size_t)k * a.ldw;
            for (int c = c_beg; c < c_end; c += 4) {
                const int n = n0 + c;
                const float4 v = *reinterpret_cast<const float4*>(arow + c);
                if (n + 3 < a.N) {
                    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};"
                                 :: "l"(wrow + n), "f"(v.x * inv), "f"(v.y * inv), "f"(v.z * inv), "f"(v.w * inv) : "memory");
                } else {
                    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) if (n + e < a.N) atomicAdd(wrow + n + e, vv[e] * inv);
                }
            }
        }
    }
}

// ---- operand conversion ------------------------------------------------------------------------------------------------
// one atomicMax per CTA (8 warps -> shared memory -> thread 0): thousands of same-address atomics serialise in L2
__device__ __forceinline__ void block_max_to_slot(float m, unsigned* slot) {
    __shared__ float wm[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float v = wm[0];
#pragma unroll
        for (int i = 1; i < 8; ++i) v = fmaxf(v, wm[i]);
        if (v > 0.f) atomicMax(slot, __float_as_uint(v));
    }
}

// largest magnitude of a (rows, C) tensor with leading dimension ld -> atomicMax on the float bits (magnitudes order like uints).
// VEC: C, ld multiples of 4 and a 16-byte aligned base (float4 loads); else scalar.
template <bool VEC>
__global__ void absmax_kernel(const float* __restrict__ x, int ld, long long rows, int C, unsigned* slot) {
    float m = 0.f;
    if (VEC) {
        const int C4 = C >> 2;
        const long long n = rows * C4;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
            const long long r = i / C4;
            const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * ld) + (i - r * C4));
            m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
        }
    } else {
        const long long n = rows * C;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
            const long long r = i / C;
            m = fmaxf(m, fabsf(x[r * ld + (i - r * C)]));
        }
    }
    block_max_to_slot(m, slot);
}
void launch_absmax(const float* x, int ld, long long rows, int C, unsigned* slot, cudaStream_t s) {
    const bool vec = (C & 3) == 0 && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    const long long n = vec ? rows * (C >> 2) : rows * C;
    const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>(592, (n + 255) / 256));
    if (vec) absmax_kernel<true><<<grid, 256, 0, s>>>(x, ld, rows, C, slot);
    else absmax_kernel<false><<<grid, 256, 0, s>>>(x, ld, rows, C, slot);
}

// (rows, C) fp32 -> planes (rows, ldp), columns >= C zero; one thread per 8 columns (one 16-byte store per plane)
__global__ void to_planes_kernel(const float* __restrict__ x, int ld, long long rows, int C, __half* __restrict__ hi,
                                 __half* __restrict__ lo, int ldp, const unsigned* slot, int vec) {
    const int g8 = ldp >> 3;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * g8) return;
    const long long r = i / g8;
    const int c = (int)(i - r * g8) * 8;
    const float s = slot_scale(slot);
    const float* p = x + r * ld + c;
    float v[8];
    if (vec && c + 8 <= C) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = (c + e < C) ? p[e] : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] *= s;
    split_store_f16<8>(v, hi + r * ldp + c, lo + r * ldp + c);
}
void launch_to_planes(const float* x, int ld, long long rows, int C, __half* hi, __half* lo, int ldp, const unsigned* slot, cudaStream_t s) {
    const int vec = ((ld & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) ? 1 : 0;
    const long long n = rows * (ldp >> 3);
    to_planes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, ld, rows, C, hi, lo, ldp, slot, vec);
}

// (B, L, C) fp32 -> transposed planes (nshift, B, C, ldt): out[j][b][c][t] = x[b][t + shift_j][c] (zero outside [0, L)).
// The tap shift runs along the contiguous (reduction) index of the weight-gradient GEMM, and TMA wants the innermost
// start coordinate 16-byte aligned (an odd shift trapped as an illegal instruction) -- so every tap gets its own, already
// shifted copy and all boxes start at multiples of 32 rows.
struct Shifts { int n; int s[3]; };
__global__ void to_planes_t_kernel(const float* __restrict__ x, int ld, int B, int L, int C, __half* __restrict__ hi,
                                   __half* __restrict__ lo, int ldt, Shifts sh, const unsigned* slot) {
    __shared__ float tile[64][33];                     // 64 time rows x 32 channels; stores are two time rows (4 bytes) per thread
    const int j = blockIdx.z / B, b = blockIdx.z - j * B, t0 = blockIdx.x * 64, c0 = blockIdx.y * 32;
    const int shift = sh.s[j];
    const float s = slot_scale(slot);
    for (int i = threadIdx.y; i < 64; i += blockDim.y) {
        const int t = t0 + i, ts = t + shift, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (t < L && ts >= 0 && ts < L && c < C) ? x[((size_t)b * L + ts) * ld + c] * s : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, t = t0 + 2 * threadIdx.x;
        if (c < C && t < ldt) {                        // ldt is a multiple of 8 and t even: the pair stays inside the row
            __half h0, l0, h1, l1;
            split_f16(tile[2 * threadIdx.x][i], h0, l0);
            split_f16(tile[2 * threadIdx.x + 1][i], h1, l1);
            const size_t o = (((size_t)j * B + b) * C + c) * ldt + t;
            *reinterpret_cast<__half2*>(hi + o) = __halves2half2(h0, h1);
            *reinterpret_cast<__half2*>(lo + o) = __halves2half2(l0, l1);
        }
    }
}

struct WTaps { const float* w[3]; };
__global__ void absmax_w_kernel(WTaps taps, int ntaps, int K, int N, int ldw, unsigned* slot) {
    const long long per = (long long)K * N, n = per * ntaps;
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int tp = (int)(i / per);
        const long long j = i - tp * per;
        const long long k = j / N;
        m = fmaxf(m, fabsf(taps.w[tp][k * ldw + (j - k * N)]));
    }
    block_max_to_slot(m, slot);
}
// W_tap[k][n] (ldw) -> K-major planes out[n][tap * Kp2 + k], n < Nrows, zero where k >= K or n >= N
__global__ void w_to_planes_kernel(WTaps taps, int K, int N, int ldw, __half* __restrict__ hi, __half* __restrict__ lo, int Kp2,
                                   int Ktot, int Nrows, const unsigned* slot) {
    __shared__ float tile[32][33];
    const int tp = blockIdx.z, k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
    const float s = slot_scale(slot);
    const float* w = taps.w[tp];
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int k = k0 + i, n = n0 + threadIdx.x;
        tile[i][threadIdx.x] = (k < K && n < N) ? w[(size_t)k * ldw + n] * s : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int n = n0 + i, k = k0 + threadIdx.x;
        if (n < Nrows && k < Kp2) {
            const size_t o = (size_t)n * Ktot + (size_t)tp * Kp2 + k;
            split_f16(tile[threadIdx.x][i], hi[o], lo[o]);
        }
    }
}

inline int roundup_i(int x, int m) { return (x + m - 1) / m * m; }

void prepare_gemm_kernel() {
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (done[dev & 63]) return;
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaFuncSetAttribute(gemm_tc_kernel): ") + cudaGetErrorString(e));
    done[dev & 63] = true;
}

int pick_bn(int N) { return std::min(256, roundup_i(N, 16)); }

void launch_gemm(const CUtensorMap m[4], GemmTcArgs& a, dim3 grid, cudaStream_t s) {
    prepare_gemm_kernel();
    // the deepest ring (<= 4 stages) that fits beside nothing else: after the main loop the ring holds the fp32 tile
    a.stages = G_MAX_STAGES;
    while (a.stages > 2 && (size_t)g_ring_bytes(a.stages, a.bn) + G_AUX + 1024 > (size_t)227 * 1024) --a.stages;
    const size_t smem = (size_t)g_ring_bytes(a.stages, a.bn) + G_AUX + 1024;
    if (a.part) gemm_tc_kernel<true><<<grid, G_THREADS, smem, s>>>(m[0], m[1], m[2], m[3], a);
    else gemm_tc_kernel<false><<<grid, G_THREADS, smem, s>>>(m[0], m[1], m[2], m[3], a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("gemm_tc_kernel launch: ") + cudaGetErrorString(e));
}

unsigned* take_slot(GemmTcWs& ws) {
    if (ws.cursor >= ws.n_slots) throw std::runtime_error("gemm_tc: out of scale slots (gemm_tc_begin_step not called?)");
    return ws.slots + ws.cursor++;
}

}  // namespace

void gemm_tc_begin_step(GemmTcWs& ws, cudaStream_t s) {
    ws.cursor = 0;
    if (ws.slots) cudaMemsetAsync(ws.slots, 0, (size_t)ws.n_slots * sizeof(unsigned), s);
}

bool conv_gemm_tc_ok(const ConvArgs& c, const GemmTcWs& ws) {
    if (!ws.slots || c.win.jptr || c.win.R != c.win.L || c.ostride != 1 || c.ooff != 0 || c.Lout != c.win.L) return false;
    if (c.ntaps < 1 || c.ntaps > 3 || (c.ldy & 3) || c.N < 1 || c.K < 1) return false;
    const size_t rows = (size_t)c.win.B * c.win.L;
    const int bn = pick_bn(c.N);
    const size_t nrows = (size_t)roundup_i(c.N, bn);
    return rows * roundup_i(c.K, 8) <= ws.a_elems && nrows * c.ntaps * roundup_i(c.K, G_BK) <= ws.b_elems;
}

// Y (+)= bias + conv(X, W) -- same contract as launch_conv_gemm's tiled path.  io (optional): a non-null slot means "this
// tensor's abs-max is already there" (the same tensor was converted earlier in this step); the slots used are returned in io.
// Returns the number of kernels launched.
int launch_conv_gemm_tc(const ConvArgs& c, GemmTcWs& ws, cudaStream_t s, GemmTcSlots* io) {
    const int B = c.win.B, L = c.win.L;
    const long long rows = (long long)B * L;
    const int ldp = roundup_i(c.K, 8), Kp2 = roundup_i(c.K, G_BK), Ktot = c.ntaps * Kp2;
    const int bn = pick_bn(c.N), n_tiles = (c.N + bn - 1) / bn, Nrows = n_tiles * bn;
    int launches = 3;
    unsigned* sa = io ? io->x : nullptr;
    unsigned* sb = io ? io->w : nullptr;
    if (!sa) { sa = take_slot(ws); launch_absmax(c.X, c.ldx, rows, c.K, sa, s); ++launches; }
    launch_to_planes(c.X, c.ldx, rows, c.K, ws.a_hi, ws.a_lo, ldp, sa, s);
    WTaps taps{};
    for (int j = 0; j < c.ntaps; ++j) taps.w[j] = c.taps[j].W;
    if (!sb) {
        sb = take_slot(ws);
        absmax_w_kernel<<<(unsigned)std::min<long long>(592, ((long long)c.ntaps * c.K * c.N + 255) / 256), 256, 0, s>>>(taps, c.ntaps, c.K, c.N, c.ldw, sb);
        ++launches;
    }
    w_to_planes_kernel<<<dim3((Kp2 + 31) / 32, (Nrows + 31) / 32, c.ntaps), dim3(32, 8), 0, s>>>(taps, c.K, c.N, c.ldw, ws.b_hi, ws.b_lo, Kp2, Ktot,
                                                                                               Nrows, sb);
    CUtensorMap m[4];
    tc_make_map3(&m[0], ws.a_hi, c.K, L, B, (uint64_t)ldp * 2, (uint64_t)L * ldp * 2, G_BK, G_BM);
    tc_make_map3(&m[1], ws.a_lo, c.K, L, B, (uint64_t)ldp * 2, (uint64_t)L * ldp * 2, G_BK, G_BM);
    tc_make_map3(&m[2], ws.b_hi, Ktot, Nrows, 1, (uint64_t)Ktot * 2, (uint64_t)Nrows * Ktot * 2, G_BK, bn);
    tc_make_map3(&m[3], ws.b_lo, Ktot, Nrows, 1, (uint64_t)Ktot * 2, (uint64_t)Nrows * Ktot * 2, G_BK, bn);
    GemmTcArgs a{};
    a.mode = 0; a.bn = bn; a.L = L; a.Lout = c.Lout; a.tiles_t = (L + G_BM - 1) / G_BM; a.ntaps = c.ntaps;
    a.kb_per_tap = Kp2 / G_BK; a.Kp2 = Kp2; a.N = c.N;
    for (int j = 0; j < c.ntaps; ++j) a.shifts[j] = c.taps[j].shift;
    a.Y = c.Y; a.ldy = c.ldy; a.bias = c.bias; a.accumulate = c.accumulate;
    a.slot_a = sa; a.slot_b = sb; a.probe = ws.probe;
    launch_gemm(m, a, dim3((unsigned)n_tiles, (unsigned)(a.tiles_t * B), 1), s);
    if (io) { io->x = sa; io->w = sb; }
    return launches;
}

bool conv_wgrad_tc_ok(const WgradArgs& w, int B, const GemmTcWs& ws) {
    if (!ws.slots || B < 1 || w.rows != (long long)B * w.L || w.ntaps < 1 || w.ntaps > 3 || (w.ldw & 3)) return false;
    const size_t ldt = (size_t)roundup_i(w.L, 8);
    return (size_t)w.ntaps * B * w.K * ldt <= ws.a_elems && (size_t)B * w.N * ldt <= ws.b_elems;
}

// The split over the batch: about `target` CTAs in all, each split a whole number of batch elements, none empty
static void wgrad_tc_split(int B, int base, int target, int& ksplit, int& nb_per_split) {
    const int k = std::max(1, std::min(B, (target + base - 1) / base));
    nb_per_split = (B + k - 1) / k;
    ksplit = (B + nb_per_split - 1) / nb_per_split;
}

// The ordered mode's fixed target: two CTAs per SM of a 132-SM H100 SXM, a constant so that the split -- and with it the
// order of the sums -- does not depend on the device
constexpr int G_ORDERED_CTAS = 264;

static int wgrad_tc_base(const WgradArgs& w) { return ((w.N + pick_bn(w.N) - 1) / pick_bn(w.N)) * ((w.K + G_BM - 1) / G_BM) * w.ntaps; }

size_t conv_wgrad_tc_ordered_floats(const WgradArgs& w, int B) {
    int ksplit, nb;
    wgrad_tc_split(B, wgrad_tc_base(w), G_ORDERED_CTAS, ksplit, nb);
    return ksplit > 1 ? (size_t)ksplit * w.ntaps * w.K * roundup_i(w.N, 4) : 0;
}

// dW[tap][k][n] += sum_rows X[b, t + shift_tap, k] dy[b, t, n] -- same contract as launch_conv_wgrad (taps contiguous:
// dW + tap * K * ldw).  io: x = slot of X, w = slot of dy (see above).  ord: the ordered mode (kernels.cuh: OrderedWs).
// Returns the number of kernels launched.
int launch_conv_wgrad_tc(const WgradArgs& w, int B, GemmTcWs& ws, cudaStream_t s, GemmTcSlots* io, const OrderedWs* ord) {
    const int L = w.L, ldt = roundup_i(L, 8);
    int launches = 3;
    unsigned* sa = io ? io->x : nullptr;
    unsigned* sb = io ? io->w : nullptr;
    if (!sa) { sa = take_slot(ws); launch_absmax(w.X, w.ldx, w.rows, w.K, sa, s); ++launches; }
    Shifts sh{}; sh.n = w.ntaps;
    for (int j = 0; j < w.ntaps; ++j) sh.s[j] = w.shifts[j];
    to_planes_t_kernel<<<dim3((ldt + 63) / 64, (w.K + 31) / 32, B * w.ntaps), dim3(32, 8), 0, s>>>(w.X, w.ldx, B, L, w.K, ws.a_hi, ws.a_lo, ldt, sh, sa);
    if (!sb) { sb = take_slot(ws); launch_absmax(w.dy, w.ldy, w.rows, w.N, sb, s); ++launches; }
    Shifts none{}; none.n = 1;
    to_planes_t_kernel<<<dim3((ldt + 63) / 64, (w.N + 31) / 32, B), dim3(32, 8), 0, s>>>(w.dy, w.ldy, B, L, w.N, ws.b_hi, ws.b_lo, ldt, none, sb);
    const int bn = pick_bn(w.N), n_tiles = (w.N + bn - 1) / bn, k_tiles = (w.K + G_BM - 1) / G_BM;
    CUtensorMap m[4];
    tc_make_map3(&m[0], ws.a_hi, L, w.K, (uint64_t)w.ntaps * B, (uint64_t)ldt * 2, (uint64_t)w.K * ldt * 2, G_BK, G_BM);
    tc_make_map3(&m[1], ws.a_lo, L, w.K, (uint64_t)w.ntaps * B, (uint64_t)ldt * 2, (uint64_t)w.K * ldt * 2, G_BK, G_BM);
    tc_make_map3(&m[2], ws.b_hi, L, w.N, B, (uint64_t)ldt * 2, (uint64_t)w.N * ldt * 2, G_BK, bn);
    tc_make_map3(&m[3], ws.b_lo, L, w.N, B, (uint64_t)ldt * 2, (uint64_t)w.N * ldt * 2, G_BK, bn);
    GemmTcArgs a{};
    a.mode = 1; a.bn = bn; a.N = w.N; a.K = w.K; a.B = B; a.tblocks = (L + G_BK - 1) / G_BK;
    const int base = n_tiles * k_tiles * w.ntaps;
    int target = G_ORDERED_CTAS;
    if (!ord) {
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        target = 2 * sms;
    }
    wgrad_tc_split(B, base, target, a.ksplit, a.nb_per_split);
    a.dW = w.dW; a.ldw = w.ldw; a.tap_stride = (long long)w.K * w.ldw;
    a.slot_a = sa; a.slot_b = sb; a.probe = ws.probe;
    // one split adds each element once: no order to fix.  The ingest probe stores nothing, so it has nothing to reduce.
    if (ord && a.ksplit > 1 && !ws.probe) {
        a.ldp = roundup_i(w.N, 4);
        const size_t need = (size_t)a.ksplit * w.ntaps * w.K * a.ldp;
        if (need > ord->part_elems)
            throw std::runtime_error("gemm_tc weight gradient: the ordered reduction needs " + std::to_string(need) +
                                     " partial floats, the workspace holds " + std::to_string(ord->part_elems));
        a.part = ord->part;
    }
    launch_gemm(m, a, dim3((unsigned)n_tiles, (unsigned)k_tiles, (unsigned)(w.ntaps * a.ksplit)), s);
    if (a.part) {
        ColSegs sg;
        sg.nseg = 1; sg.s[0] = ColSeg{w.dW, 0, a.ldp, w.N, w.ldw};
        launch_ordered_colsum<float>(a.part, a.ksplit, (long long)w.ntaps * w.K * a.ldp, sg, s);
        ++launches;
    }
    if (io) { io->x = sa; io->w = sb; }
    return launches;
}

}  // namespace dctts
