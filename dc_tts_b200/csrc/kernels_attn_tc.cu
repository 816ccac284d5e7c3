// kernels_attn_tc.cu -- the dot-product attention (reference networks.py:126-155) as ONE
// wgmma kernel: S = Q K^T / sqrt(d) -> window mask -> softmax -> argmax -> A V -> [A V ; Q],
// alignments written transposed.  One CTA per (128 query rows, utterance): a TMA producer
// warp and two consumer warpgroups of 64 query rows each.
//
//   GEMM 1  S[128 x 192]  = Q[128 x 256] . K^T        (keys padded 180 -> 192 by TMA zero fill)
//   softmax on the register accumulators, four threads per query row (quad shuffles);
//           the probabilities are written back to shared memory as split-fp16 planes in the
//           128B-swizzled K-major layout the tensor core reads (no global round trip)
//   GEMM 2  C[128 x 256]  = P[128 x 192] . V          (V pre-transposed to [d][keys] planes)
// Both GEMMs use the split-fp16 three-pass scheme (hi*hi + hi*lo + lo*hi, fp32 accumulate):
// the argmax of these probabilities is fed back into the next decode step, so the scores
// need fp32-grade accuracy.  Shared memory (160 KB) is reused: GEMM 1's two 80 KB pipeline
// stages become P (96 KB) and one 64 KB V^T stage.
#include "kernels_tc.cuh"
#include "tc_ptx.cuh"

#include <algorithm>
#include <stdexcept>
#include <string>

namespace dctts {

using namespace ptx;

constexpr int AT_THREADS = 384;
constexpr int AT_NP = 192;                        // padded key count (3 x 64)
constexpr int AT_D = 256;                         // head width (hp.d)
constexpr int AT_Q_PLANE = 128 * 64 * 2;          // 16 KB: 128 query rows x 64 channels fp16
constexpr int AT_K_PLANE = AT_NP * 64 * 2;        // 24 KB
constexpr int AT_STAGE1 = 2 * AT_Q_PLANE + 2 * AT_K_PLANE;   // 80 KB
constexpr int AT_P_PLANE = 3 * AT_Q_PLANE;        // 48 KB: 3 key blocks of [128 x 64]
constexpr int AT_VT_PLANE = AT_D * 64 * 2;        // 32 KB: 256 channels x 64 keys
constexpr int AT_SMEM_MAIN = 2 * AT_STAGE1;       // 160 KB

__global__ void __launch_bounds__(AT_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap mapQ_hi, const __grid_constant__ CUtensorMap mapQ_lo,
                    const __grid_constant__ CUtensorMap mapK_hi, const __grid_constant__ CUtensorMap mapK_lo,
                    const __grid_constant__ CUtensorMap mapV_hi, const __grid_constant__ CUtensorMap mapV_lo,
                    const AttnTcArgs a) {
    extern __shared__ uint8_t at_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AT_SMEM_MAIN);
    uint64_t* full_bar = bars;            // [2]
    uint64_t* empty_bar = bars + 2;       // [2]
    uint64_t* s_full = bars + 4;          // GEMM 1 done in both consumer warpgroups: its stages are free
    uint64_t* vt_full = bars + 6;
    uint64_t* vt_empty = bars + 7;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int b = blockIdx.y, t0 = blockIdx.x * 128;
    const int T = a.T, N = a.N;

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&mapQ_hi); prefetch_tmap(&mapQ_lo); prefetch_tmap(&mapK_hi); prefetch_tmap(&mapK_lo);
        prefetch_tmap(&mapV_hi); prefetch_tmap(&mapV_lo);
        for (int s = 0; s < 2; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        mbar_init(s_full, 2); mbar_init(vt_full, 1); mbar_init(vt_empty, 2);
        fence_mbar_init();
    }
    __syncthreads();

    uint8_t* p_hi = smem;                          // [3][128 rows][128 B]
    uint8_t* p_lo = smem + AT_P_PLANE;
    uint8_t* vt_st = smem + 2 * AT_P_PLANE;        // V^T hi (32 KB) | lo (32 KB)

    if (warp == 0) {
        // =========================== TMA producer ===========================
        if (lane == 0) {
            for (int kb = 0; kb < AT_D / 64; ++kb) {
                const int s = kb & 1;
                mbar_wait(&empty_bar[s], ((uint32_t)(kb >> 1) & 1u) ^ 1u);
                mbar_expect_tx(&full_bar[s], AT_STAGE1);
                uint8_t* st = smem + (size_t)s * AT_STAGE1;
                tma_load_3d(&mapQ_hi, &full_bar[s], st, kb * 64, t0, b);
                tma_load_3d(&mapQ_lo, &full_bar[s], st + AT_Q_PLANE, kb * 64, t0, b);
                tma_load_3d(&mapK_hi, &full_bar[s], st + 2 * AT_Q_PLANE, kb * 64, 0, b);
                tma_load_3d(&mapK_lo, &full_bar[s], st + 2 * AT_Q_PLANE + AT_K_PLANE, kb * 64, 0, b);
            }
            mbar_wait(s_full, 0);                  // GEMM 1 has consumed its stages: the memory is free
            for (int kb = 0; kb < AT_NP / 64; ++kb) {
                mbar_wait(vt_empty, ((uint32_t)kb & 1u) ^ 1u);
                mbar_expect_tx(vt_full, 2 * AT_VT_PLANE);
                tma_load_3d(&mapV_hi, vt_full, vt_st, kb * 64, 0, b);
                tma_load_3d(&mapV_lo, vt_full, vt_st + AT_VT_PLANE, kb * 64, 0, b);
            }
        }
        __syncwarp();
        return;
    }
    if (wg == 0) return;                           // warps 1-3: no role
    // =========================== consumers: query rows 64 * mh .. +64 of the tile ===========================
    const int mh = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    const int rq = mh * 64 + (warp & 3) * 16 + (lane >> 2);        // fragment rows rq, rq + 8; columns 8 i + 2 (lane & 3) + {0, 1}
    // ---- GEMM 1: S = Q K^T, 64 x 192 per warpgroup (three 64-key chunks) ----
    float sacc[3][32];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) sacc[j][i] = 0.f;
    for (int kb = 0; kb < AT_D / 64; ++kb) {
        const int s = kb & 1;
        mbar_wait(&full_bar[s], (uint32_t)(kb >> 1) & 1u);
        const uint32_t st = smem_u32(smem + (size_t)s * AT_STAGE1);
        const uint64_t dQ_hi = gmma_desc_kmajor<128>(st + mh * 64 * 128), dQ_lo = gmma_desc_kmajor<128>(st + AT_Q_PLANE + mh * 64 * 128);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t adv = (uint64_t)(k * 2);
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const uint64_t dK_hi = gmma_desc_kmajor<128>(st + 2 * AT_Q_PLANE + j * 64 * 128);
                const uint64_t dK_lo = gmma_desc_kmajor<128>(st + 2 * AT_Q_PLANE + AT_K_PLANE + j * 64 * 128);
                wgmma_f16<4>(sacc[j], dQ_hi + adv, dK_hi + adv, (kb | k) != 0);
                wgmma_f16<4>(sacc[j], dQ_hi + adv, dK_lo + adv, 1u);
                wgmma_f16<4>(sacc[j], dQ_lo + adv, dK_hi + adv, 1u);
            }
        }
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int j = 0; j < 3; ++j) wg_fence_regs(sacc[j]);
        if (leader) mbar_arrive(&empty_bar[s]);
    }
    if (leader) mbar_arrive(s_full);
    named_sync(1, 256);                            // both warpgroups are done with GEMM 1's stages: P may overwrite them

    // ---- softmax over the live keys, four threads per query row (quad shuffles) ----
    int n_lo = 0, n_hi = N;
    if (a.pma) {                                   // monotonic window [p, p + win) (networks.py:141-147)
        const int p = __ldg(a.pma + b);
        n_lo = min(max(p, 0), N - 1);
        n_hi = min(n_lo + a.win_size, N);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {                  // the thread's two rows
        const int r = rq + 8 * h, t = t0 + r;
        const bool row_ok = t < T;
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = j * 64 + i * 8 + 2 * (lane & 3) + e;
                    if (n >= n_lo && n < n_hi) mx = fmaxf(mx, sacc[j][i * 4 + 2 * h + e] * a.scale);
                }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = j * 64 + i * 8 + 2 * (lane & 3) + e;
                    if (n >= n_lo && n < n_hi) sum += expf(sacc[j][i * 4 + 2 * h + e] * a.scale - mx);
                }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        // probabilities -> split planes in shared memory (128B-swizzled K-major, GEMM 2's A operand), alignments, argmax
        float best = -1.f; int besti = 0;
        float* al = (a.align && row_ok) ? a.align + (size_t)b * N * T + t : nullptr;
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float p2[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = j * 64 + i * 8 + 2 * (lane & 3) + e;
                    float p = 0.f;                 // masked keys are exactly 0 in the reference (exp underflow)
                    if (n >= n_lo && n < n_hi) p = expf(sacc[j][i * 4 + 2 * h + e] * a.scale - mx) / sum;
                    if (p > best) { best = p; besti = n; }
                    if (al && n < N) al[(size_t)n * T] = p;
                    p2[e] = p;
                }
                const __half h0 = __float2half_rn(p2[0]), h1 = __float2half_rn(p2[1]);
                const __half l0 = __float2half_rn(p2[0] - __half2float(h0)), l1 = __float2half_rn(p2[1] - __half2float(h1));
                const int off = j * AT_Q_PLANE + r * 128 + ((i ^ (r & 7)) << 4) + 4 * (lane & 3);
                *reinterpret_cast<__half2*>(p_hi + off) = __halves2half2(h0, h1);
                *reinterpret_cast<__half2*>(p_lo + off) = __halves2half2(l0, l1);
            }
        // argmax over the quad: the first key of the largest probability, as a sequential scan finds it
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
        }
        if (row_ok && a.maxatt && (lane & 3) == 0) a.maxatt[(size_t)b * T + t] = (long long)besti;
    }
    fence_proxy_async_smem();                      // generic-proxy stores -> visible to the tensor core
    named_sync(1, 256);

    // ---- GEMM 2: context = P V, 64 x 256 per warpgroup (four 64-channel chunks) ----
    float cacc[4][32];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) cacc[j][i] = 0.f;
    for (int kb = 0; kb < AT_NP / 64; ++kb) {
        mbar_wait(vt_full, (uint32_t)kb & 1u);
        const uint64_t dP_hi = gmma_desc_kmajor<128>(smem_u32(p_hi + kb * AT_Q_PLANE + mh * 64 * 128));
        const uint64_t dP_lo = gmma_desc_kmajor<128>(smem_u32(p_lo + kb * AT_Q_PLANE + mh * 64 * 128));
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t adv = (uint64_t)(k * 2);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint64_t dV_hi = gmma_desc_kmajor<128>(smem_u32(vt_st + j * 64 * 128));
                const uint64_t dV_lo = gmma_desc_kmajor<128>(smem_u32(vt_st + AT_VT_PLANE + j * 64 * 128));
                wgmma_f16<4>(cacc[j], dP_hi + adv, dV_hi + adv, (kb | k) != 0);
                wgmma_f16<4>(cacc[j], dP_hi + adv, dV_lo + adv, 1u);
                wgmma_f16<4>(cacc[j], dP_lo + adv, dV_hi + adv, 1u);
            }
        }
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int j = 0; j < 4; ++j) wg_fence_regs(cacc[j]);
        if (leader) mbar_arrive(vt_empty);
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
                    const __half vh0 = __float2half_rn(v.x), vh1 = __float2half_rn(v.y);
                    const __half qh0 = __float2half_rn(q.x), qh1 = __float2half_rn(q.y);
                    __half* dh = a.Rpl.hi + row * a.Rpl.ld;
                    __half* dl = a.Rpl.lo + row * a.Rpl.ld;
                    *reinterpret_cast<__half2*>(dh + c) = __halves2half2(vh0, vh1);
                    *reinterpret_cast<__half2*>(dl + c) = __halves2half2(__float2half_rn(v.x - __half2float(vh0)), __float2half_rn(v.y - __half2float(vh1)));
                    *reinterpret_cast<__half2*>(dh + AT_D + c) = __halves2half2(qh0, qh1);
                    *reinterpret_cast<__half2*>(dl + AT_D + c) = __halves2half2(__float2half_rn(q.x - __half2float(qh0)), __float2half_rn(q.y - __half2float(qh1)));
                }
            }
    }
}

// K (B,N,d) and V (B,N,d) fp32 (leading dimension ld) -> K planes (B,N,d) and V^T planes (B,d,192)
__global__ void attn_kv_planes_kernel(const float* __restrict__ K, int ldk, const float* __restrict__ V, int ldv,
                                      Planes kp, Planes vtp, int B, int N, int d) {
    const long long total = (long long)B * AT_NP * d;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % d);
        const int n = (int)((i / d) % AT_NP);
        const int b = (int)(i / ((long long)d * AT_NP));
        float kv = 0.f, vv = 0.f;
        if (n < N) { kv = K[((size_t)b * N + n) * ldk + c]; vv = V[((size_t)b * N + n) * ldv + c]; }
        if (n < N) {
            __half h = __float2half_rn(kv);
            kp.hi[((size_t)b * N + n) * kp.ld + c] = h;
            kp.lo[((size_t)b * N + n) * kp.ld + c] = __float2half_rn(kv - __half2float(h));
        }
        __half h = __float2half_rn(vv);
        vtp.hi[((size_t)b * d + c) * vtp.ld + n] = h;                 // keys >= N are written as zeros
        vtp.lo[((size_t)b * d + c) * vtp.ld + n] = __float2half_rn(vv - __half2float(h));
    }
}

void launch_attn_kv_planes(const float* K, int ldk, const float* V, int ldv, Planes kp, Planes vtp, int B, int N, int d,
                           cudaStream_t s) {
    const long long total = (long long)B * AT_NP * d;
    const int grid = (int)std::min<long long>((total + 255) / 256, 4096);
    attn_kv_planes_kernel<<<grid, 256, 0, s>>>(K, ldk, V, ldv, kp, vtp, B, N, d);
}

int attn_tc_padded_keys() { return AT_NP; }

void launch_attention_tc(const Planes& Q, const Planes& K, const Planes& Vt, const AttnTcArgs& a, int B, cudaStream_t s) {
    if (a.d != AT_D || a.N > AT_NP) throw std::runtime_error("attention_tc: unsupported d / N");
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
    tc_make_act_map(&mq_h, Q.hi, a.d, Q.ld, a.T, B, 128, 1, 64);
    tc_make_act_map(&mq_l, Q.lo, a.d, Q.ld, a.T, B, 128, 1, 64);
    tc_make_act_map(&mk_h, K.hi, a.d, K.ld, a.N, B, AT_NP, 1, 64);     // rows N..191 out of bounds -> zeros
    tc_make_act_map(&mk_l, K.lo, a.d, K.ld, a.N, B, AT_NP, 1, 64);
    tc_make_act_map(&mv_h, Vt.hi, AT_NP, Vt.ld, a.d, B, AT_D, 1, 64);  // (keys, channels, batch), box {64 keys, 256 channels}
    tc_make_act_map(&mv_l, Vt.lo, AT_NP, Vt.ld, a.d, B, AT_D, 1, 64);
    dim3 grid((a.T + 127) / 128, B);
    attention_tc_kernel<<<grid, AT_THREADS, smem, s>>>(mq_h, mq_l, mk_h, mk_l, mv_h, mv_l, a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("attention_tc launch: ") + cudaGetErrorString(e));
}

}  // namespace dctts
