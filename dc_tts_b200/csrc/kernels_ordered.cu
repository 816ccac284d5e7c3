// kernels_ordered.cu -- the training step's sums in a fixed order (option "train_deterministic"; DESIGN.md 8e,
// "Deterministic training").  One pattern everywhere: every CTA writes its partial sums to a workspace with plain stores, in
// a layout fixed by the shape alone, and ordered_colsum_kernel adds the partials in a fixed order and does the single
// read-modify-write of the destination.  The split counts depend on the shape only, never on the device, so the same
// inputs give the same bits on any handle, at any workspace capacity, after any history.
//   ordered_colsum_kernel            the reduction (float for gradients, double for the loss sums)
//   train_block_bwd_ordered_kernel   the block backward; within a CTA the 8 warps' values are combined in warp order
//   conv_wgrad_part_kernel           the fp32 weight gradient, one partial dW per row split
//   train_loss_ordered_kernel, attn_loss_ordered_kernel   the losses on a fixed grid, one partial row per CTA
//   embed_bwd_ordered_kernel         the embedding gradient: one thread per (id, channel) sums the text positions in order
// The wgmma weight gradient (kernels_gemm_tc.cu) stores its split tiles to the same workspace and reduces with the same kernel.
#include "kernels.cuh"
#include "kernels_train.cuh"
#include "numerics.cuh"

#include <algorithm>

namespace dctts {

namespace {

void check_room(size_t need, size_t have, const char* what) {
    if (need > have)
        throw std::runtime_error(std::string(what) + ": the ordered reduction needs " + std::to_string(need) +
                                 " partial elements, the workspace holds " + std::to_string(have));
}

}  // namespace

// ------------------------------------------------------------------------------------ the ordered reduction
// 32 columns x 8 lanes per CTA: lane y adds partials y, y + 8, y + 16, ... in index order, then lane 0 adds the eight lane
// sums in lane order onto the destination.
template <typename T>
__global__ void __launch_bounds__(256) ordered_colsum_kernel(const T* __restrict__ part, long long nparts, long long width, const ColSegs sg) {
    __shared__ T red[8][33];
    const long long col = (long long)blockIdx.x * 32 + threadIdx.x;
    T v = 0;
    if (col < width)
        for (long long p = threadIdx.y; p < nparts; p += 8) v += part[p * width + col];
    red[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.y != 0 || col >= width) return;
    T t = red[0][threadIdx.x];
#pragma unroll
    for (int j = 1; j < 8; ++j) t += red[j][threadIdx.x];
    ColSeg g = sg.s[0];
#pragma unroll
    for (int j = 1; j < 5; ++j)                        // constant indices: a dynamic one would copy the params to the stack
        if (j < sg.nseg && col >= sg.s[j].col0) g = sg.s[j];
    const long long i = col - g.col0, r = i / g.n;
    const int c = (int)(i - r * g.n);
    if (c < g.w) { T* d = static_cast<T*>(g.dst) + r * g.ld + c; *d += t; }
}

template <typename T> void launch_ordered_colsum(const T* part, long long nparts, long long width, const ColSegs& sg, cudaStream_t s) {
    ordered_colsum_kernel<T><<<(unsigned)((width + 31) / 32), dim3(32, 8), 0, s>>>(part, nparts, width, sg);
}
template void launch_ordered_colsum<float>(const float*, long long, long long, const ColSegs&, cudaStream_t);
template void launch_ordered_colsum<double>(const double*, long long, long long, const ColSegs&, cudaStream_t);

// ------------------------------------------------------------------------------------ block backward
// The values of train_block_bwd_kernel (kernels_train.cu); where it adds with shared-memory atomics, every warp stores the
// value to its own slice of a stage in shared memory, [quantity][warp][C], and after each row slot (one row per warp) the
// CTA adds the slices, warp 0 first, onto its accumulator.  At the end the accumulator is one partial row of `width`
// floats, [dg1 C][db1 C]([dg2 C][db2 C])[dbias nconv], stored to part[blockIdx.x].  A warp past the last row computes on
// the slot's first row, stores nothing and stages zeros.
// Dynamic shared memory: the accumulator (width floats) and the stage (4 x BWD_WARPS x C floats, 2 x for mode 0).

// acc[j] += sum over warps of stage[q][warp][c], j = q C + c < nq C, after a barrier; ends with one
__device__ __forceinline__ void stage_flush(const float* __restrict__ stage, float* __restrict__ acc, int nq, int C) {
    __syncthreads();
    for (int j = threadIdx.x; j < nq * C; j += blockDim.x) {
        const int q = j / C, c = j - q * C;
        float v = acc[j];
#pragma unroll
        for (int w = 0; w < BWD_WARPS; ++w) v += stage[(q * BWD_WARPS + w) * C + c];
        acc[j] = v;
    }
    __syncthreads();
}

template <int MAXV, bool HC>
__global__ void __launch_bounds__(BWD_WARPS * 32) train_block_bwd_ordered_kernel(const BlockBwdArgs a, float* __restrict__ part) {
    extern __shared__ float sm[];
    const int C = a.C, nconv = a.mode == 1 ? 2 * C : C, nln = a.mode == 1 ? 4 * C : 2 * C, width = nln + nconv;
    float* stage = sm + width;
    for (int i = threadIdx.x; i < width; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* st0 = stage + (0 * BWD_WARPS + warp) * C; float* st1 = stage + (1 * BWD_WARPS + warp) * C;
    float* st2 = stage + (2 * BWD_WARPS + warp) * C; float* st3 = stage + (3 * BWD_WARPS + warp) * C;
    for (int rr = 0; rr < BWD_ROWS_PER_WARP; ++rr) {
        const long long row0 = (long long)blockIdx.x * BWD_WARPS * BWD_ROWS_PER_WARP + rr;      // warp 0's row: the slot's first
        if (row0 >= a.rows) break;                                                            // CTA-uniform
        const long long own = ((long long)blockIdx.x * BWD_WARPS + warp) * BWD_ROWS_PER_WARP + rr;
        const bool valid = own < a.rows;
        const float vm = valid ? 1.f : 0.f;
        const long long row = valid ? own : row0;
        const float* y = a.pre + row * a.ldy;
        const float* go = a.gout + row * a.ldg;
        float* dyo = a.dy + row * a.ldy;
        float yh1[MAXV], dz1[MAXV], dy1[MAXV];
        float r1;
        ln_fwd_half<MAXV>(y, C, lane, yh1, r1);
        if (!HC || a.mode == 0) {
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                const int c = lane + 32 * i;
                float g = 0.f;
                if (c < C) {
                    g = go[c] * keep_mul((uint32_t)(row * C + c), a.drop);
                    const float z = yh1[i] * __ldg(a.g1 + c) + __ldg(a.b1 + c);
                    if (a.act == 1 && !(z > 0.f)) g = 0.f;
                    st0[c] = vm * (g * yh1[i]); st1[c] = vm * g;
                }
                dz1[i] = g;
            }
            ln_bwd_half<MAXV>(yh1, dz1, a.g1, C, lane, r1, dy1);
            stage_flush(stage, sm, 2, C);
#pragma unroll
            for (int i = 0; i < MAXV; ++i) { const int c = lane + 32 * i; if (c < C) { if (valid) dyo[c] = dy1[i]; st0[c] = vm * dy1[i]; } }
            stage_flush(stage, sm + nln, 1, C);
        } else {
            float yh2[MAXV], dz2[MAXV], dy2[MAXV];
            float r2;
            ln_fwd_half<MAXV>(y + C, C, lane, yh2, r2);
            const float* x = a.X + row * a.ldx;
            float* gi = a.gin + row * a.ldg;
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                const int c = lane + 32 * i;
                float d1 = 0.f, d2 = 0.f;
                if (c < C) {
                    const float g = go[c] * keep_mul((uint32_t)(row * C + c), a.drop);
                    const float h1 = sigmoid_acc(yh1[i] * __ldg(a.g1 + c) + __ldg(a.b1 + c));
                    const float h2 = yh2[i] * __ldg(a.g2 + c) + __ldg(a.b2 + c);
                    d1 = g * (h2 - x[c]) * h1 * (1.0f - h1);
                    d2 = g * h1;
                    if (valid) gi[c] = g * (1.0f - h1);                            // highway path; the data gradient adds to it
                    st0[c] = vm * (d1 * yh1[i]); st1[c] = vm * d1;
                    st2[c] = vm * (d2 * yh2[i]); st3[c] = vm * d2;
                }
                dz1[i] = d1; dz2[i] = d2;
            }
            ln_bwd_half<MAXV>(yh1, dz1, a.g1, C, lane, r1, dy1);
            ln_bwd_half<MAXV>(yh2, dz2, a.g2, C, lane, r2, dy2);
            stage_flush(stage, sm, 4, C);
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                const int c = lane + 32 * i;
                if (c < C) {
                    if (valid) { dyo[c] = dy1[i]; dyo[C + c] = dy2[i]; }
                    st0[c] = vm * dy1[i]; st1[c] = vm * dy2[i];
                }
            }
            stage_flush(stage, sm + nln, 2, C);
        }
    }
    float* prow = part + (size_t)blockIdx.x * width;
    for (int i = threadIdx.x; i < width; i += blockDim.x) prow[i] = sm[i];     // the last stage_flush ended with a barrier
}

size_t block_bwd_ordered_floats(long long rows, int C, int mode) {
    const long long ctas = (rows + BWD_WARPS * BWD_ROWS_PER_WARP - 1) / (BWD_WARPS * BWD_ROWS_PER_WARP);
    return (size_t)ctas * (size_t)((mode == 1 ? 6 : 3) * C);
}

template <int MAXV, bool HC>
int launch_train_block_bwd_ordered(const BlockBwdArgs& a, const OrderedWs& o, cudaStream_t s) {
    const int rows_per_cta = BWD_WARPS * BWD_ROWS_PER_WARP;
    const long long grid = (a.rows + rows_per_cta - 1) / rows_per_cta;
    const int C = a.C, nconv = a.mode == 1 ? 2 * C : C, nln = a.mode == 1 ? 4 * C : 2 * C, width = nln + nconv;
    check_room(block_bwd_ordered_floats(a.rows, C, a.mode), o.part_elems, "train_block_bwd");
    const size_t smem = (size_t)(width + (a.mode == 1 ? 4 : 2) * BWD_WARPS * C) * sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(train_block_bwd_ordered_kernel<MAXV, HC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            cudaGetLastError();
            throw std::runtime_error("train_block_bwd (ordered): " + std::to_string(smem) + " bytes of shared memory: " + cudaGetErrorString(e));
        }
    }
    train_block_bwd_ordered_kernel<MAXV, HC><<<(unsigned)grid, BWD_WARPS * 32, smem, s>>>(a, o.part);
    ColSegs sg;
    auto seg = [&](float* dst, int col0, int n) { sg.s[sg.nseg++] = ColSeg{dst, col0, n, n, n}; };
    seg(a.dg1, 0, C); seg(a.db1, C, C);
    if (a.mode == 1) { seg(a.dg2, 2 * C, C); seg(a.db2, 3 * C, C); }
    seg(a.dbias, nln, nconv);
    launch_ordered_colsum<float>(o.part, grid, width, sg, s);
    return 2;
}
template int launch_train_block_bwd_ordered<4, true>(const BlockBwdArgs&, const OrderedWs&, cudaStream_t);
template int launch_train_block_bwd_ordered<8, true>(const BlockBwdArgs&, const OrderedWs&, cudaStream_t);
template int launch_train_block_bwd_ordered<16, true>(const BlockBwdArgs&, const OrderedWs&, cudaStream_t);
template int launch_train_block_bwd_ordered<32, true>(const BlockBwdArgs&, const OrderedWs&, cudaStream_t);
template int launch_train_block_bwd_ordered<33, true>(const BlockBwdArgs&, const OrderedWs&, cudaStream_t);
template int launch_train_block_bwd_ordered<65, false>(const BlockBwdArgs&, const OrderedWs&, cudaStream_t);

// ------------------------------------------------------------------------------------ fp32 weight gradient
// conv_wgrad_kernel's tile, stored to part[split][tap][K][ldp] (ldp = N rounded up to 4) instead of added to dW
__global__ void __launch_bounds__(256) conv_wgrad_part_kernel(const WgradArgs a, float* __restrict__ part, int ldp) {
    __shared__ __align__(16) float Xs[16][64 + 4];
    __shared__ __align__(16) float Ds[16][64 + 4];
    const int n0 = blockIdx.x * 64, k0 = blockIdx.y * 64;
    const int tap = blockIdx.z / a.nsplit, split = blockIdx.z - tap * a.nsplit;
    const int shift = tap == 0 ? a.shifts[0] : tap == 1 ? a.shifts[1] : a.shifts[2];
    const long long r_begin = (long long)split * a.rows_per_split, r_end = min((long long)a.rows, r_begin + a.rows_per_split);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4];
    wgrad_tile(a, n0, k0, shift, r_begin, r_end, Xs, Ds, acc);
    float* P = part + ((size_t)split * a.ntaps + tap) * a.K * ldp;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int k = k0 + ty * 4 + i;
        if (k >= a.K) continue;
        const int n = n0 + tx * 4;
        if (n < ldp) *reinterpret_cast<float4*>(P + (size_t)k * ldp + n) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
}

// The default split, min(64, rows / 512), capped so that about 1024 tiles run: enough CTAs for the device, and partials of at
// most (1024 + tiles) 64 x 64 tiles.  With one split every element has one contributor and the default kernel is ordered.
int conv_wgrad_ordered_splits(const WgradArgs& w) {
    const long long tiles = (long long)((w.N + 63) / 64) * ((w.K + 63) / 64) * w.ntaps;
    const long long by_rows = std::max<long long>(1, std::min<long long>(64, w.rows / 512));
    return (int)std::max<long long>(1, std::min(by_rows, (1024 + tiles - 1) / tiles));
}

size_t conv_wgrad_ordered_floats(const WgradArgs& w) {
    const int nsplit = conv_wgrad_ordered_splits(w);
    return nsplit > 1 ? (size_t)nsplit * w.ntaps * w.K * ((w.N + 3) / 4 * 4) : 0;
}

int launch_conv_wgrad_ordered(const WgradArgs& a, const OrderedWs& o, cudaStream_t s) {
    const int ldp = (a.N + 3) / 4 * 4;
    check_room((size_t)a.nsplit * a.ntaps * a.K * ldp, o.part_elems, "conv_wgrad");
    dim3 grid((a.N + 63) / 64, (a.K + 63) / 64, a.ntaps * a.nsplit);
    conv_wgrad_part_kernel<<<grid, 256, 0, s>>>(a, o.part, ldp);
    ColSegs sg;
    sg.nseg = 1; sg.s[0] = ColSeg{a.dW, 0, ldp, a.N, a.ldw};                   // rows tap * K + k of dW (taps contiguous)
    launch_ordered_colsum<float>(o.part, a.nsplit, (long long)a.ntaps * a.K * ldp, sg, s);
    return 2;
}

// ------------------------------------------------------------------------------------ losses
// 256 threads sum their elements in index order, the warps by a fixed shuffle tree, thread 0 the 8 warps in order
__device__ __forceinline__ double block_sum_ordered(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int k = 0; k < 8; ++k) t += red[k];
    return t;
}

__global__ void __launch_bounds__(256) train_loss_ordered_kernel(const float* __restrict__ logits, int ldl, const float* __restrict__ target,
                                                                 float* __restrict__ dlogits, int ldg, double* __restrict__ part, long long n, int C) {
    __shared__ double red[2][8];
    double l1 = 0.0, bce = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float e1, e2;
        loss_element(logits, ldl, target, dlogits, ldg, i, n, C, e1, e2);
        l1 += e1; bce += e2;
    }
    const double a = block_sum_ordered(l1, red[0]), b = block_sum_ordered(bce, red[1]);
    if (threadIdx.x == 0) { part[2 * blockIdx.x] = a; part[2 * blockIdx.x + 1] = b; }
}

int launch_train_loss_ordered(const float* logits, int ldl, const float* target, float* dlogits, int ldg, double* sums, long long rows,
                              int C, const OrderedWs& o, cudaStream_t s) {
    const long long n = rows * C;
    const int grid = (int)std::min<long long>(ORD_LOSS_CTAS, (n + 255) / 256);
    check_room(2 * (size_t)grid, o.dpart_elems, "train_loss");
    train_loss_ordered_kernel<<<grid, 256, 0, s>>>(logits, ldl, target, dlogits, ldg, o.dpart, n, C);
    ColSegs sg;
    sg.nseg = 1; sg.s[0] = ColSeg{sums, 0, 2, 2, 2};
    launch_ordered_colsum<double>(o.dpart, grid, 2, sg, s);
    return 2;
}

__global__ void __launch_bounds__(256) attn_loss_ordered_kernel(const float* __restrict__ align, const float* __restrict__ gts, int ld_gts,
                                                                double* __restrict__ part, int B, int N, int T, int n_lim, int t_lim) {
    __shared__ double red[8];
    const long long total = (long long)B * N * T;
    double v = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long nt = i % ((long long)N * T);
        const int n = (int)(nt / T), t = (int)(nt - (long long)n * T);
        if (n < n_lim && t < t_lim) v += fabsf(align[i] * gts[(size_t)n * ld_gts + t]);
    }
    const double a = block_sum_ordered(v, red);
    if (threadIdx.x == 0) part[blockIdx.x] = a;
}

int launch_attn_loss_ordered(const float* align, const float* gts, int ld_gts, double* sums, int B, int N, int T, int n_lim, int t_lim,
                             const OrderedWs& o, cudaStream_t s) {
    const long long n = (long long)B * N * T;
    const int grid = (int)std::min<long long>(ORD_LOSS_CTAS, (n + 255) / 256);
    check_room((size_t)grid, o.dpart_elems, "attn_loss");
    attn_loss_ordered_kernel<<<grid, 256, 0, s>>>(align, gts, ld_gts, o.dpart, B, N, T, n_lim, t_lim);
    ColSegs sg;
    sg.nseg = 1; sg.s[0] = ColSeg{sums + 2, 0, 1, 1, 1};
    launch_ordered_colsum<double>(o.dpart, grid, 1, sg, s);
    return 2;
}

// ------------------------------------------------------------------------------------ embedding backward
// CTA = one id of [1, vocab), thread = channels c, c + 128, ...: the text positions with that id in index order.  The table is
// small (vocab x e) and a batch's text short, so no workspace: the sums run where the gradient is read.
__global__ void __launch_bounds__(128) embed_bwd_ordered_kernel(const int* __restrict__ ids, const float* __restrict__ g,
                                                                float* __restrict__ dtable, int rows, int e) {
    const int id = blockIdx.x + 1;
    for (int c = threadIdx.x; c < e; c += blockDim.x) {
        float v = 0.f;
        bool any = false;
        for (int r = 0; r < rows; ++r)
            if (__ldg(ids + r) == id) { v += g[(size_t)r * e + c]; any = true; }
        if (any) dtable[(size_t)id * e + c] += v;
    }
}

int launch_embed_bwd_ordered(const int* ids, const float* g, float* dtable, int rows, int e, int vocab, cudaStream_t s) {
    if (vocab < 2) throw std::runtime_error("embed_bwd (ordered): the vocabulary has no id past 0");
    embed_bwd_ordered_kernel<<<vocab - 1, 128, 0, s>>>(ids, g, dtable, rows, e);
    return 1;
}

}  // namespace dctts
