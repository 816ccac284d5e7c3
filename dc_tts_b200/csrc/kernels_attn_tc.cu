// kernels_attn_tc.cu -- the dot-product attention (reference networks.py:126-155) as ONE
// wgmma kernel: S = Q K^T / sqrt(d) -> window mask -> softmax -> argmax -> A V -> [A V ; Q],
// alignments written transposed.  One CTA per (64 query rows, utterance): one consumer
// warpgroup, which holds C (128 registers) beside one S block, and a TMA producer warp.
// Any key count N: the keys are visited in blocks of 64 (nb = ceil(N / 64), the last one
// zero-filled by TMA past N), and S is never held for more than one block:
//
//   pass 1  per key block: S[64 x 64] = Q[64 x 256] . K_blk^T     -> row max
//   pass 2  per key block: S again                                 -> per-thread sum of exp(s - max)
//   pass 3  per key block: S again -> probabilities, alignments, argmax, P block in shared memory
//           (split-fp16 planes, 128B-swizzled K-major: GEMM 2's A operand) -> C[64 x 256] += P_blk . V_blk
//
// Each S accumulator sees the wgmma sequence d-slab, k-step, hi*hi, hi*lo, lo*hi in all three
// passes, each C accumulator key block, k-step and the same three products, and the sums and
// the argmax scan visit the keys in (block, i, e) order: the same arithmetic as holding all of S
// in registers, which the three 64-key blocks of N <= 192 would allow.  With the monotonic window only the blocks that hold a
// live key are computed; the others are exactly 0 in every output.
// Both GEMMs use the split-fp16 three-pass scheme (hi*hi + hi*lo + lo*hi, fp32 accumulate):
// the argmax of these probabilities is fed back into the next decode step, so the scores
// need fp32-grade accuracy.
// Shared memory does not depend on N (176 KB): Q stays resident (4 d-slabs x hi/lo, 64 KB),
// the P block (16 KB), and a 6-stage ring of 16 KB stages carrying K slabs (64 keys x 64
// channels) and, in pass 3, V^T chunks (64 channels x 64 keys), both as hi | lo.
#include "kernels_tc.cuh"
#include "numerics.cuh"
#include "tc_ptx.cuh"

#include <algorithm>
#include <stdexcept>
#include <string>

namespace dctts {

using namespace ptx;

constexpr int AT_THREADS = 160;                   // warpgroup 0: consumer; warp 4: TMA producer
constexpr int AT_D = 256;                         // head width (hp.d)
constexpr int AT_ROWS = 64;                       // query rows per CTA
constexpr int AT_Q_PLANE = AT_ROWS * 64 * 2;      // 8 KB: 64 query rows x 64 channels fp16
constexpr int AT_Q_BYTES = 2 * (AT_D / 64) * AT_Q_PLANE;   // 64 KB: every d-slab, hi and lo
constexpr int AT_P_PLANE = AT_ROWS * 64 * 2;      // 8 KB: 64 query rows x 64 keys fp16
constexpr int AT_HALF = 64 * 64 * 2;              // 8 KB: one plane of a ring stage
constexpr int AT_STAGE = 2 * AT_HALF;             // 16 KB: hi | lo
constexpr int AT_STAGES = 6;
constexpr int AT_SMEM_MAIN = AT_Q_BYTES + 2 * AT_P_PLANE + AT_STAGES * AT_STAGE;   // 176 KB

// the key blocks holding a live key of [n_lo, n_hi): [jb0, jb1)
__device__ __forceinline__ void attn_live_blocks(const AttnTcArgs& a, int b, int& n_lo, int& n_hi, int& jb0, int& jb1) {
    n_lo = 0; n_hi = a.N;
    if (a.pma) {                                   // monotonic window [p, p + win) (networks.py:141-147)
        const int p = __ldg(a.pma + b);
        n_lo = min(max(p, 0), a.N - 1);
        n_hi = min(n_lo + a.win_size, a.N);
    }
    jb0 = n_lo >> 6;
    jb1 = n_hi > n_lo ? ((n_hi - 1) >> 6) + 1 : jb0;
}

__global__ void __launch_bounds__(AT_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap mapQ_hi, const __grid_constant__ CUtensorMap mapQ_lo,
                    const __grid_constant__ CUtensorMap mapK_hi, const __grid_constant__ CUtensorMap mapK_lo,
                    const __grid_constant__ CUtensorMap mapV_hi, const __grid_constant__ CUtensorMap mapV_lo,
                    const AttnTcArgs a) {
    extern __shared__ uint8_t at_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* q_st = smem;                                  // [d-slab][hi, lo][64 rows][128 B]
    uint8_t* p_hi = smem + AT_Q_BYTES;                     // [64 rows][128 B]
    uint8_t* p_lo = p_hi + AT_P_PLANE;
    uint8_t* ring = p_lo + AT_P_PLANE;                     // [stage][hi, lo][64 rows][128 B]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AT_SMEM_MAIN);
    uint64_t* full_bar = bars;                     // [AT_STAGES]
    uint64_t* empty_bar = bars + AT_STAGES;        // [AT_STAGES]
    uint64_t* q_full = bars + 2 * AT_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y, t0 = blockIdx.x * AT_ROWS;
    const int T = a.T, N = a.N;
    const int nb = (N + 63) >> 6;
    int n_lo, n_hi, jb0, jb1;
    attn_live_blocks(a, b, n_lo, n_hi, jb0, jb1);

    if (warp == 4 && lane == 0) {
        prefetch_tmap(&mapQ_hi); prefetch_tmap(&mapQ_lo); prefetch_tmap(&mapK_hi); prefetch_tmap(&mapK_lo);
        prefetch_tmap(&mapV_hi); prefetch_tmap(&mapV_lo);
        for (int s = 0; s < AT_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
        mbar_init(q_full, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 4) {
        // =========================== TMA producer: Q once, then the ring in the consumer's order ===========================
        if (lane == 0) {
            mbar_expect_tx(q_full, AT_Q_BYTES);
            for (int kb = 0; kb < AT_D / 64; ++kb) {
                tma_load_3d(&mapQ_hi, q_full, q_st + (2 * kb) * AT_Q_PLANE, kb * 64, t0, b);
                tma_load_3d(&mapQ_lo, q_full, q_st + (2 * kb + 1) * AT_Q_PLANE, kb * 64, t0, b);
            }
            uint32_t it = 0;
            auto next_stage = [&](uint32_t bytes) {
                const int s = (int)(it % AT_STAGES);
                mbar_wait(&empty_bar[s], ((it / AT_STAGES) & 1u) ^ 1u);
                mbar_expect_tx(&full_bar[s], bytes);
                ++it;
                return s;
            };
            for (int pass = 0; pass < 3; ++pass)
                for (int jb = jb0; jb < jb1; ++jb) {
                    for (int kb = 0; kb < AT_D / 64; ++kb) {           // K slab: keys jb*64.., channels kb*64..
                        const int s = next_stage(AT_STAGE);
                        uint8_t* st = ring + (size_t)s * AT_STAGE;
                        tma_load_3d(&mapK_hi, &full_bar[s], st, kb * 64, jb * 64, b);
                        tma_load_3d(&mapK_lo, &full_bar[s], st + AT_HALF, kb * 64, jb * 64, b);
                    }
                    if (pass == 2)
                        for (int j = 0; j < AT_D / 64; ++j) {          // V^T chunk: channels j*64.., keys jb*64..
                            const int s = next_stage(AT_STAGE);
                            uint8_t* st = ring + (size_t)s * AT_STAGE;
                            tma_load_3d(&mapV_hi, &full_bar[s], st, jb * 64, j * 64, b);
                            tma_load_3d(&mapV_lo, &full_bar[s], st + AT_HALF, jb * 64, j * 64, b);
                        }
                }
        }
        __syncwarp();
        return;
    }
    // =========================== consumer warpgroup ===========================
    const bool leader = threadIdx.x == 0;
    const int rq = warp * 16 + (lane >> 2);       // fragment rows rq, rq + 8; columns 8 i + 2 (lane & 3) + {0, 1}
    uint32_t it = 0;                               // ring position, in step with the producer
    mbar_wait(q_full, 0);

    // S for the ring's next key block, 64 x 64: one ring stage per d-slab, the previous slab's MMAs still in flight
    auto gemm_s = [&](float (&sacc)[32]) {
        for (int kb = 0; kb < AT_D / 64; ++kb) {
            const int s = (int)(it % AT_STAGES);
            mbar_wait(&full_bar[s], (it / AT_STAGES) & 1u);
            const uint32_t st = smem_u32(ring + (size_t)s * AT_STAGE);
            const uint64_t dQ_hi = gmma_desc_kmajor<128>(smem_u32(q_st + (2 * kb) * AT_Q_PLANE));
            const uint64_t dQ_lo = gmma_desc_kmajor<128>(smem_u32(q_st + (2 * kb + 1) * AT_Q_PLANE));
            const uint64_t dK_hi = gmma_desc_kmajor<128>(st), dK_lo = gmma_desc_kmajor<128>(st + AT_HALF);
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t adv = (uint64_t)(k * 2);
                wgmma_f16<4>(sacc, dQ_hi + adv, dK_hi + adv, (kb | k) != 0);
                wgmma_f16<4>(sacc, dQ_hi + adv, dK_lo + adv, 1u);
                wgmma_f16<4>(sacc, dQ_lo + adv, dK_hi + adv, 1u);
            }
            wg_commit();
            if (kb > 0) {
                wg_wait<1>();
                if (leader) mbar_arrive(&empty_bar[(it - 1) % AT_STAGES]);
            }
            ++it;
        }
        wg_wait<0>();
        wg_fence_regs(sacc);
        if (leader) mbar_arrive(&empty_bar[(it - 1) % AT_STAGES]);
    };

    float sacc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
    // ---- pass 1: row max over the live keys (four threads per query row, quad shuffles) ----
    float mx[2] = {-INFINITY, -INFINITY};
    for (int jb = jb0; jb < jb1; ++jb) {
        gemm_s(sacc);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = jb * 64 + i * 8 + 2 * (lane & 3) + e;
                    if (n >= n_lo && n < n_hi) mx[h] = fmaxf(mx[h], sacc[i * 4 + 2 * h + e] * a.scale);
                }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    // ---- pass 2: the softmax denominators ----
    float sum[2] = {0.f, 0.f};
    for (int jb = jb0; jb < jb1; ++jb) {
        gemm_s(sacc);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = jb * 64 + i * 8 + 2 * (lane & 3) + e;
                    if (n >= n_lo && n < n_hi) sum[h] += expf(sacc[i * 4 + 2 * h + e] * a.scale - mx[h]);
                }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
    }

    // ---- pass 3: probabilities -> alignments, argmax, P block; context = P V, 64 x 256 ----
    float cacc[4][32];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) cacc[j][i] = 0.f;
    float best[2] = {-1.f, -1.f};
    int besti[2] = {0, 0};
    const uint64_t dP_hi = gmma_desc_kmajor<128>(smem_u32(p_hi));
    const uint64_t dP_lo = gmma_desc_kmajor<128>(smem_u32(p_lo));
    for (int jb = 0; jb < nb; ++jb) {
        const bool live = jb >= jb0 && jb < jb1;
        if (live) gemm_s(sacc);
#pragma unroll
        for (int h = 0; h < 2; ++h) {              // the thread's two rows
            const int r = rq + 8 * h, t = t0 + r;
            float* al = (a.align && t < T) ? a.align + (size_t)b * N * T + t : nullptr;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float p2[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = jb * 64 + i * 8 + 2 * (lane & 3) + e;
                    float p = 0.f;                 // masked keys are exactly 0 in the reference (exp underflow)
                    if (live && n >= n_lo && n < n_hi) p = expf(sacc[i * 4 + 2 * h + e] * a.scale - mx[h]) / sum[h];
                    if (p > best[h]) { best[h] = p; besti[h] = n; }
                    if (al && n < N) al[(size_t)n * T] = p;
                    p2[e] = p;
                }
                if (live) {
                    __half2 h, l;
                    split_f16x2(make_float2(p2[0], p2[1]), h, l);
                    const int off = r * 128 + ((i ^ (r & 7)) << 4) + 4 * (lane & 3);
                    *reinterpret_cast<__half2*>(p_hi + off) = h;
                    *reinterpret_cast<__half2*>(p_lo + off) = l;
                }
            }
        }
        if (!live) continue;
        fence_proxy_async_smem();                  // generic-proxy stores -> visible to the tensor core
        named_sync(1, 128);
        for (int j = 0; j < 4; ++j) {              // one V^T chunk (64 channels) per ring stage
            const int s = (int)(it % AT_STAGES);
            mbar_wait(&full_bar[s], (it / AT_STAGES) & 1u);
            const uint32_t st = smem_u32(ring + (size_t)s * AT_STAGE);
            const uint64_t dV_hi = gmma_desc_kmajor<128>(st), dV_lo = gmma_desc_kmajor<128>(st + AT_HALF);
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t adv = (uint64_t)(k * 2);
                wgmma_f16<4>(cacc[j], dP_hi + adv, dV_hi + adv, (jb != jb0 || k != 0) ? 1u : 0u);
                wgmma_f16<4>(cacc[j], dP_hi + adv, dV_lo + adv, 1u);
                wgmma_f16<4>(cacc[j], dP_lo + adv, dV_hi + adv, 1u);
            }
            wg_commit();
            if (j > 0) {
                wg_wait<1>();
                if (leader) mbar_arrive(&empty_bar[(it - 1) % AT_STAGES]);
            }
            ++it;
        }
        wg_wait<0>();
#pragma unroll
        for (int j = 0; j < 4; ++j) wg_fence_regs(cacc[j]);
        if (leader) mbar_arrive(&empty_bar[(it - 1) % AT_STAGES]);
        named_sync(1, 128);                        // the P block is read: the next block may overwrite it
    }
    // argmax over the quad: the first key of the largest probability, as a sequential scan finds it
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best[h], o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti[h], o);
            if (ob > best[h] || (ob == best[h] && oi < besti[h])) { best[h] = ob; besti[h] = oi; }
        }
        const int t = t0 + rq + 8 * h;
        if (t < T && a.maxatt && (lane & 3) == 0) a.maxatt[(size_t)b * T + t] = (long long)besti[h];
    }

    // ---- R = [context ; Q] straight from the fragments ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int t = t0 + rq + 8 * h;
        if (t >= T) continue;
        const size_t row = (size_t)b * T + t;
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int c = j * 64 + i * 8 + 2 * (lane & 3);
                const float2 v = make_float2(cacc[j][i * 4 + 2 * h], cacc[j][i * 4 + 2 * h + 1]);
                const float2 q = __ldg(reinterpret_cast<const float2*>(a.Q + row * a.ldq + c));
                *reinterpret_cast<float2*>(a.R + row * a.ldr + c) = v;
                *reinterpret_cast<float2*>(a.R + row * a.ldr + AT_D + c) = q;
                if (a.Rpl.hi) {
                    __half* dh = a.Rpl.hi + row * a.Rpl.ld;
                    __half* dl = a.Rpl.lo + row * a.Rpl.ld;
                    split_f16x2(v, *reinterpret_cast<__half2*>(dh + c), *reinterpret_cast<__half2*>(dl + c));
                    split_f16x2(q, *reinterpret_cast<__half2*>(dh + AT_D + c), *reinterpret_cast<__half2*>(dl + AT_D + c));
                }
            }
    }
}

// K (B,N,d) and V (B,N,d) fp32 (leading dimension ld) -> K planes (B,N,d) and V^T planes (B,d,NP), NP = vtp.ld >= N keys
// (attn_tc_padded_keys), keys >= N written as zeros
__global__ void attn_kv_planes_kernel(const float* __restrict__ K, int ldk, const float* __restrict__ V, int ldv,
                                      Planes kp, Planes vtp, int B, int N, int d) {
    const int NP = vtp.ld;
    const long long total = (long long)B * NP * d;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % d);
        const int n = (int)((i / d) % NP);
        const int b = (int)(i / ((long long)d * NP));
        float kv = 0.f, vv = 0.f;
        if (n < N) { kv = K[((size_t)b * N + n) * ldk + c]; vv = V[((size_t)b * N + n) * ldv + c]; }
        if (n < N) split_f16(kv, kp.hi[((size_t)b * N + n) * kp.ld + c], kp.lo[((size_t)b * N + n) * kp.ld + c]);
        split_f16(vv, vtp.hi[((size_t)b * d + c) * vtp.ld + n], vtp.lo[((size_t)b * d + c) * vtp.ld + n]);   // keys >= N: zeros
    }
}

void launch_attn_kv_planes(const float* K, int ldk, const float* V, int ldv, Planes kp, Planes vtp, int B, int N, int d,
                           cudaStream_t s) {
    if (vtp.ld < attn_tc_padded_keys(N)) throw std::runtime_error("attn_kv_planes: V^T planes narrower than the padded key count");
    const long long total = (long long)B * vtp.ld * d;
    const int grid = (int)std::min<long long>((total + 255) / 256, 4096);
    attn_kv_planes_kernel<<<grid, 256, 0, s>>>(K, ldk, V, ldv, kp, vtp, B, N, d);
}

int attn_tc_padded_keys(int N) { return (N + 63) / 64 * 64; }

void launch_attention_tc(const Planes& Q, const Planes& K, const Planes& Vt, const AttnTcArgs& a, int B, cudaStream_t s) {
    if (a.d != AT_D || a.N < 1) throw std::runtime_error("attention_tc: unsupported d / N");
    if (Vt.ld < attn_tc_padded_keys(a.N)) throw std::runtime_error("attention_tc: V^T planes narrower than the padded key count");
    static bool attr_set_dev[64] = {};      // per device (the attribute is per device, not per process)
    int dev = 0;
    cudaGetDevice(&dev);
    bool& attr_set = attr_set_dev[dev & 63];
    const size_t smem = AT_SMEM_MAIN + 128 + 1024;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) throw std::runtime_error(std::string("cudaFuncSetAttribute(attention_tc): ") + cudaGetErrorString(e));
        attr_set = true;
    }
    CUtensorMap mq_h, mq_l, mk_h, mk_l, mv_h, mv_l;
    tc_make_act_map(&mq_h, Q.hi, a.d, Q.ld, a.T, B, AT_ROWS, 1, 64);   // rows >= T read zeros
    tc_make_act_map(&mq_l, Q.lo, a.d, Q.ld, a.T, B, AT_ROWS, 1, 64);
    tc_make_act_map(&mk_h, K.hi, a.d, K.ld, a.N, B, 64, 1, 64);        // {64 channels, 64 keys}; keys >= N read zeros
    tc_make_act_map(&mk_l, K.lo, a.d, K.ld, a.N, B, 64, 1, 64);
    tc_make_act_map(&mv_h, Vt.hi, Vt.ld, Vt.ld, a.d, B, 64, 1, 64);    // (keys, channels, batch), box {64 keys, 64 channels}
    tc_make_act_map(&mv_l, Vt.lo, Vt.ld, Vt.ld, a.d, B, 64, 1, 64);
    dim3 grid((a.T + AT_ROWS - 1) / AT_ROWS, B);
    attention_tc_kernel<<<grid, AT_THREADS, smem, s>>>(mq_h, mq_l, mk_h, mk_l, mv_h, mv_l, a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("attention_tc launch: ") + cudaGetErrorString(e));
}

}  // namespace dctts
