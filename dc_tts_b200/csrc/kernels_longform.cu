// kernels_longform.cu -- the long-form join (DESIGN.md section 4e): the decoded pieces of each text, written one after
// another into that text's mel sequence with rows of silence between them.  One CTA per piece p of text k = text[p]:
//   offset_p    sum over the pieces q of text k before p of (min(max(len[q], 0), T) + pause[q])   (the prefix sum)
//   rows        out[k, offset_p + t] = Y[p, t] for t < len[p], then pause[p] rows of `silence`
//   last piece  out_len[k] = offset_p + len[p] (its pause is 0), and rows [out_len[k], T_out) of out[k] are zeros
// Every CTA sums its own prefix from the lengths the decode left on the device, so the join needs no host copy of them.
// Latency-bound: a few hundred rows of n_mels floats per CTA.
#include "kernels.cuh"

namespace dctts {

namespace {

constexpr int JOIN_THREADS = 256;

__global__ void __launch_bounds__(JOIN_THREADS) join_rows_kernel(const JoinArgs a) {
    __shared__ long long s_off;
    const int p = blockIdx.x, tid = threadIdx.x;
    const int k = a.text[p], first = a.first[k], last = a.first[k + 1] - 1;
    if (tid == 0) {
        long long off = 0;
        for (int q = first; q < p; ++q) off += min(max(a.len[q], 0), a.T) + a.pause[q];
        s_off = off;
    }
    __syncthreads();
    const long long off = s_off;
    const int n = min(max(a.len[p], 0), a.T), C = a.C;
    float* o = a.out + ((size_t)k * a.T_out + off) * C;
    const float* y = a.Y + (size_t)p * a.T * C;
    const long long live = (long long)n * C, filled = live + (long long)a.pause[p] * C;
    for (long long i = tid; i < live; i += JOIN_THREADS) o[i] = y[i];
    for (long long i = live + tid; i < filled; i += JOIN_THREADS) o[i] = a.silence;
    if (p == last) {
        const long long end = off + n, tail = ((long long)a.T_out - end) * C;
        for (long long i = live + tid; i < live + tail; i += JOIN_THREADS) o[i] = 0.f;
        if (tid == 0) a.out_len[k] = (int)end;
    }
}

}  // namespace

void launch_join_rows(const JoinArgs& a, cudaStream_t s) {
    join_rows_kernel<<<a.P, JOIN_THREADS, 0, s>>>(a);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("join_rows_kernel launch failed: ") + cudaGetErrorString(e));
}

}  // namespace dctts
