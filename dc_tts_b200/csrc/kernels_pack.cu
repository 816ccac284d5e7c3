// kernels_pack.cu -- the weight packers: the live fp32 layer weights W ([tap][cin][ldw], the buffers the optimiser updates)
// into the split-fp16 planes of the wgmma block kernel (kernels_tc.cu) and the per-rank weight stream of the persistent
// decode (kernels_decode.cu).  Both run at commit and at every dctts_refresh_synthesis, so a trained handle synthesises
// from exactly the bytes a fresh handle holding the same variables would.  The host supplies the geometry, which depends
// on shapes only, and the power-of-two scales, from the abs-max this file's reduction computes.
//   weight_absmax_kernel   max |W| of every layer in one launch (order-independent: bit-identical to a serial scan)
//   pack_tc_kernel         one element of the K-major planes [nrows][Ktot] per thread, in pack order (api_params.cu)
//   pack_decode_kernel     one (rank, k row, slice column) of a decode block per thread: the fp32 GEMV layout and, for
//                          the receptive-field blocks, the split-fp16 MMA slabs
// The scaled value is formed with __fmul_rn so that no multiply-add contraction changes the rounding of the split.
#include "kernels.cuh"
#include "kernels_decode.cuh"
#include "numerics.cuh"

namespace dctts {

// ------------------------------------------------------------------------------------ abs-max
// maxbits[e] (float bits; zeroed by the caller) = max over the n[e] floats at W[e] of |x|.  NaNs are skipped, as std::max
// does when the running maximum is its first argument.  Non-negative floats order as their bit patterns.
__global__ void weight_absmax_kernel(const __grid_constant__ PackMaxTable t, unsigned* __restrict__ maxbits) {
    const float* W = t.W[blockIdx.y];
    const long long n = t.n[blockIdx.y];
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = fabsf(W[i]);
        if (v > m) m = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(maxbits + blockIdx.y, __float_as_uint(m));
}

void launch_weight_absmax(const PackMaxTable& t, unsigned* maxbits_dev, cudaStream_t s) {
    if (t.count <= 0) return;
    weight_absmax_kernel<<<dim3(64, t.count), 256, 0, s>>>(t, maxbits_dev);
}

// ------------------------------------------------------------------------------------ wgmma block planes
// Row `row` of the planes is accumulator column a = row % bn of cluster CTA i = row / bn; column k = tap * cin_pad + ci.
// mode 0 conv: W column `row` (rows >= cout are zero).  mode 1 hc: the first `half` rows of a CTA are gate channels
// i*half + a, the rest the info channels of the same index.  mode 2 transposed conv: k-tap 0 reads x[t] (W0 on the first
// half, W1 on the second), k-tap 1 reads x[t-1] (W2 on the first half, zeros on the second).
__global__ void pack_tc_kernel(TcPackArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)a.nrows * a.Ktot) return;
    const int row = (int)(i / a.Ktot), k = (int)(i % a.Ktot);
    const int tap = k / a.cin_pad, ci = k % a.cin_pad;
    float v = 0.f;
    if (ci < a.cin) {
        const int c = row / a.bn, r = row % a.bn;
        const bool second = r >= a.half;
        const int col = c * a.half + (r % a.half);
        const float* W = a.W;
        if (a.mode == 0) v = row < a.cout ? W[((size_t)tap * a.cin + ci) * a.ldw + row] : 0.f;
        else if (a.mode == 1) v = W[((size_t)tap * a.cin + ci) * a.ldw + (second ? a.cout + col : col)];
        else if (tap == 0) v = W[((size_t)(second ? 1 : 0) * a.cin + ci) * a.ldw + col];
        else v = second ? 0.f : W[((size_t)2 * a.cin + ci) * a.ldw + col];
        v = __fmul_rn(v, a.scale);
    }
    split_f16(v, a.hi[i], a.lo[i]);
}

void launch_pack_tc(const TcPackArgs& a, cudaStream_t s) {
    const long long n = (long long)a.nrows * a.Ktot;
    pack_tc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a);
}

// ------------------------------------------------------------------------------------ persistent decode stream
// Thread (r, k, n): rank r, k row k = tap * cinp + ci of the block (chunk q = k / krows, row kc = k % krows in it), slice
// column n.  A chunk is 8 warp regions of kr8 = krows / 8 rows; 32-column slices are pair-split per 8-k block
// [column parity][k-group][column pair][4 k] (gemv_warp32), narrower ones [k/4][column][4].  hc blocks: slice columns
// [0, cs) are gate channels r*cs.., [cs, 2cs) the info channels of the same index; conv blocks: cs columns, then zeros.
// The stream is zeroed before the first block is packed: rows ci >= cin and the zero columns are not written.
// Receptive-field blocks (scale > 0): the same rows as MMA slabs of 16 k, [plane hi | lo][k8 group][column][8 halfs].
__global__ void pack_decode_kernel(DecPackArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)DEC_NC * a.K * a.ns) return;
    const int n = (int)(i % a.ns), k = (int)(i / a.ns % a.K), r = (int)(i / ((long long)a.ns * a.K));
    const int q = k / a.krows, kc = k % a.krows, tap = k / a.cinp, ci = k % a.cinp;
    const int col = a.kind ? (n < a.cs ? r * a.cs + n : a.cout + r * a.cs + (n - a.cs)) : (n < a.cs ? r * a.cs + n : -1);
    const bool live = col >= 0 && ci < a.cin;
    const float w = live ? a.W[((size_t)tap * a.cin + ci) * a.ldw + col] : 0.f;
    float* rank = a.stream + (size_t)r * a.stream_len;
    const size_t chunk = (size_t)q * a.krows * a.ns;
    if (live) {
        const int kr8 = a.krows / 8, wr = kc / kr8, kk = kc % kr8;
        const size_t idx = a.ns == 32 ? (size_t)(kk / 8) * 256 + ((size_t)((n & 1) * 2 + (kk / 4) % 2) * 16 + (n >> 1)) * 4 + (kk % 4)
                                      : ((size_t)(kk / 4) * a.ns + n) * 4 + (kk % 4);
        rank[a.off + chunk + (size_t)wr * kr8 * a.ns + idx] = w;
    }
    if (a.scale > 0.f) {
        __half* d16 = reinterpret_cast<__half*>(rank + a.off16 + chunk);
        const int slab = kc / 16, k16 = kc % 16, grp = k16 / 8, e8 = k16 % 8;
        const size_t base = (size_t)slab * 32 * a.ns;                    // halfs per slab = 2 planes * 2 groups * ns * 8
        const size_t idx = ((size_t)grp * a.ns + n) * 8 + e8;
        split_f16(__fmul_rn(w, a.scale), d16[base + idx], d16[base + (size_t)2 * a.ns * 8 + idx]);
    }
}

void launch_pack_decode(const DecPackArgs& a, cudaStream_t s) {
    const long long n = (long long)DEC_NC * a.K * a.ns;
    pack_decode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a);
}

}  // namespace dctts
