// kernels_align.cu -- the aligner's search (DESIGN.md section 4d): the best monotonic path through the teacher-forced
// attention of each utterance, one CTA per utterance.
//   cost        c[n, t] = log(double(max(A[n, t], 1e-30f)))        (the floor in float32, everything after in float64)
//   paths       one character n_t per frame t < T_b: 0 <= n_0 <= w - 1, 0 <= n_t - n_{t-1} <= w - 1, n_{T_b - 1} = e_b --
//               exactly the window paths the decode can follow (frame t runs under the window n_{t-1}, n_t lies in it)
//   recurrence  D[n, 0] = c[n, 0];  D[n, t] = c[n, t] + max_{s in [0, w-1]} D[n - s, t - 1], the smaller step s on a tie
//   band        only cells that can be reached and can still reach e_b:
//               max(0, e_b - (w-1)(T_b-1-t)) <= n <= min(e_b, (w-1)(t+1))
// Two D rows of e_b + 1 doubles live in shared memory as a ping-pong; the step taken into every cell of the band is one
// byte in the back-pointer workspace (global memory).  After the last frame one thread walks back from (e_b, T_b - 1).
#include "kernels.cuh"

namespace dctts {

namespace {

constexpr int ALIGN_THREADS = 256;

__global__ void __launch_bounds__(ALIGN_THREADS) align_search_kernel(const AlignArgs a) {
    extern __shared__ double D[];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int Tb = a.meta[b], e = a.meta[a.B + b];
    const int T = a.T, N = a.N, w1 = a.win - 1;
    const float* __restrict__ A = a.A + (size_t)b * N * T;
    unsigned char* bp = a.bp + (size_t)b * T * N;
    int* chars = a.chars + (size_t)b * T;
    int* path = a.path + (size_t)b * T;
    int* dur = a.durations + (size_t)b * N;
    // what the walk back does not write; the frame loop's barrier orders these stores before it
    for (int n = tid; n < N; n += ALIGN_THREADS) dur[n] = 0;
    for (int t = Tb + tid; t < T; t += ALIGN_THREADS) { chars[t] = -1; path[t] = -1; }

    double* cur = D;
    double* prev = D + (e + 1);
    for (int t = 0; t < Tb; ++t) {
        const int lo = max(0, e - w1 * (Tb - 1 - t)), hi = min(e, w1 * (t + 1));
        const int plo = max(0, e - w1 * (Tb - t)), phi = min(e, w1 * t);    // the band at t - 1
        for (int n = lo + tid; n <= hi; n += ALIGN_THREADS) {
            const double c = log((double)fmaxf(__ldg(A + (size_t)n * T + t), 1e-30f));
            if (t == 0) { cur[n] = c; continue; }
            // predecessors n - s inside the previous band: s in [max(0, n - phi), min(w - 1, n - plo)], never empty
            const int s0 = max(0, n - phi), s1 = min(w1, n - plo);
            double best = prev[n - s0];
            int bs = s0;
            for (int s = s0 + 1; s <= s1; ++s) {
                const double v = prev[n - s];
                if (v > best) { best = v; bs = s; }
            }
            cur[n] = c + best;
            bp[(size_t)t * N + n] = (unsigned char)bs;
        }
        __syncthreads();
        double* x = cur; cur = prev; prev = x;
    }
    if (tid != 0) return;
    a.score[b] = prev[e];
    int n = e, run = 0;
    for (int t = Tb - 1; t >= 0; --t) {
        const int m = t > 0 ? n - (int)bp[(size_t)t * N + n] : -1;     // n_{t-1}: the window of frame t
        chars[t] = n;
        path[t] = t > 0 ? m : 0;
        ++run;
        if (m != n) { dur[n] = run; run = 0; }
        n = m;
    }
}

}  // namespace

void launch_align_search(const AlignArgs& a, int max_end, cudaStream_t s) {
    const size_t smem = 2 * (size_t)(max_end + 1) * sizeof(double);
    cudaError_t e = cudaFuncSetAttribute(align_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        align_search_kernel<<<a.B, ALIGN_THREADS, smem, s>>>(a);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) throw std::runtime_error(std::string("align_search_kernel launch failed: ") + cudaGetErrorString(e));
}

}  // namespace dctts
