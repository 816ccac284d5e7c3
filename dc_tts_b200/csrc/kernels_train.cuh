// kernels_train.cuh -- device code shared by the training step's default kernels (kernels_train.cu) and their ordered
// counterparts (kernels_ordered.cu, option "train_deterministic"): the LayerNorm halves of the block backward, the
// weight-gradient tile and one element of the mel / magnitude losses.  Each ordered kernel computes the same values as its
// default twin; only how the sums are combined differs.
#pragma once
#include "kernels.cuh"
#include "numerics.cuh"

namespace dctts {

constexpr int BWD_WARPS = 8;
constexpr int BWD_ROWS_PER_WARP = 4;

// LayerNorm backward for one half held in registers.  yhat = (y - mean) rstd, z = yhat g + b.
//   dy = rstd (dyh - mean(dyh) - yhat mean(dyh yhat)),  dyh = dz g
template <int MAXV>
__device__ __forceinline__ void ln_bwd_half(const float (&yhat)[MAXV], const float (&dz)[MAXV], const float* __restrict__ gam,
                                            int C, int lane, float rstd, float (&dy)[MAXV]) {
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = lane + 32 * i;
        if (c < C) { const float t = dz[i] * __ldg(gam + c); dy[i] = t; s1 += t; s2 = fmaf(t, yhat[i], s2); }
        else dy[i] = 0.f;
    }
    s1 = warp_sum(s1) / (float)C; s2 = warp_sum(s2) / (float)C;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) dy[i] = rstd * (dy[i] - s1 - yhat[i] * s2);
}

template <int MAXV>
__device__ __forceinline__ void ln_fwd_half(const float* __restrict__ y, int C, int lane, float (&yhat)[MAXV], float& rstd) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) { const int c = lane + 32 * i; yhat[i] = c < C ? y[c] : 0.f; s += yhat[i]; }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) { const int c = lane + 32 * i; const float d = c < C ? yhat[i] - mean : 0.f; yhat[i] = d; q = fmaf(d, d, q); }
    rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + 1e-12f);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) yhat[i] *= rstd;
}

// One 64 x 64 tile of dW[tap] = sum over rows [r_begin, r_end) of X[b, t + shift, k] dy[b, t, n], 256 threads, 4 x 4
// outputs each: acc[i][j] is (k0 + 4 ty + i, n0 + 4 tx + j), ty = tid / 16, tx = tid % 16.
__device__ __forceinline__ void wgrad_tile(const WgradArgs& a, int n0, int k0, int shift, long long r_begin, long long r_end,
                                           float (&Xs)[16][64 + 4], float (&Ds)[16][64 + 4], float (&acc)[4][4]) {
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;               // 16 x 16 threads, 4 x 4 outputs each
    const int lr = tid >> 4, lq = (tid & 15) * 4;         // loader: row lr (0..15), 4 consecutive columns at lq
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (long long r0 = r_begin; r0 < r_end; r0 += 16) {
        const long long row = r0 + lr;
        float4 xv = make_float4(0.f, 0.f, 0.f, 0.f), dv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < r_end) {
            const int b = (int)(row / a.L), t = (int)(row - (long long)b * a.L), ts = t + shift;
            const int k = k0 + lq, n = n0 + lq;
            if (ts >= 0 && ts < a.L && k < a.K) {
                const float* p = a.X + ((size_t)b * a.L + ts) * a.ldx + k;
                if (k + 3 < a.K) xv = __ldg(reinterpret_cast<const float4*>(p));
                else { xv.x = p[0]; if (k + 1 < a.K) xv.y = p[1]; if (k + 2 < a.K) xv.z = p[2]; }
            }
            if (n < a.N) dv = __ldg(reinterpret_cast<const float4*>(a.dy + row * a.ldy + n));     // N, ldy multiples of 4
        }
        __syncthreads();
        *reinterpret_cast<float4*>(&Xs[lr][lq]) = xv;
        *reinterpret_cast<float4*>(&Ds[lr][lq]) = dv;
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const float4 xa = *reinterpret_cast<const float4*>(&Xs[r][ty * 4]);
            const float4 db = *reinterpret_cast<const float4*>(&Ds[r][tx * 4]);
            const float av[4] = {xa.x, xa.y, xa.z, xa.w}, bv[4] = {db.x, db.y, db.z, db.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
    }
}

// Element i of the mel / magnitude losses: |Y - m| and BCE(logit, m) returned, dlogits = (sign(Y-m) Y (1-Y) + (Y - m)) / n
// stored.  logits (rows, C) with leading dimension ldl, targets dense (rows, C), dlogits (rows, C) with leading dimension ldg.
__device__ __forceinline__ void loss_element(const float* __restrict__ logits, int ldl, const float* __restrict__ target,
                                             float* __restrict__ dlogits, int ldg, long long i, long long n, int C, float& l1, float& bce) {
    const long long row = i / C;
    const int c = (int)(i - row * C);
    const float x = logits[row * ldl + c], m = target[i];
    const float y = sigmoid_acc(x);
    const float d = y - m;
    l1 = fabsf(d);
    bce = fmaxf(x, 0.f) - x * m + log1pf(expf(-fabsf(x)));
    const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    dlogits[row * ldg + c] = (sg * y * (1.0f - y) + d) / (float)n;
}

}  // namespace dctts
