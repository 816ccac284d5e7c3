// kernels_mcd.cu -- mel-cepstral distortion along a DTW alignment (DESIGN.md section 8h): one CTA per pair of mel
// sequences X[b, :nx_b] and Y[b, :ny_b] (dB-normalised, as utils.get_spectrograms writes them).
//   cepstrum    a_m = (ln 10 / 20) (max_db x_m - max_db + ref_db),  c_k = sum_m a_m D[k, m],  k = 1 .. K
//               (D the orthonormal DCT-II matrix; c_0, the energy, is left out)
//   local cost  d(i, j) = (10 / ln 10) sqrt(2 sum_k (cx_ik - cy_jk)^2)
//   recurrence  D(0, 0) = d(0, 0);  D(i, j) = d(i, j) + min(D(i-1, j-1), D(i-1, j), D(i, j-1)), ties to the first of
//               those three (strict comparisons); the path ends at (nx_b - 1, ny_b - 1)
//   outputs     mcd[b] = D(nx_b - 1, ny_b - 1) / P_b, pairs[b] = P_b (the cells on the path), optionally the path
// Everything after the float32 input is float64.  The first phase writes both sequences' cepstra, to shared memory when
// they fit there and otherwise to a global workspace read back through L2; the second sweeps the anti-diagonals
// i + j = d, three of them in shared memory (indexed by i), one barrier per diagonal.  The step taken into every cell is
// one byte in the back-pointer workspace, stored diagonal by diagonal so that a diagonal's stores are contiguous.  After
// the last diagonal one thread walks the path back from the end.
#include "kernels.cuh"

namespace dctts {

namespace {

constexpr int MCD_THREADS = 256;

// cells of the diagonals 0 .. d-1 of an nx x ny grid: where diagonal d starts in the back-pointer layout
__device__ __forceinline__ long long diag_start(long long d, long long nx, long long ny) {
    const long long s1 = d <= nx ? d * (d + 1) / 2 : nx * (nx + 1) / 2 + (d - nx) * nx;
    const long long s2 = d <= ny ? 0 : (d - ny) * (d - ny + 1) / 2;
    return s1 - s2;
}

__global__ void __launch_bounds__(MCD_THREADS) mcd_dtw_kernel(const McdArgs a) {
    extern __shared__ double sm[];
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long* meta = a.meta + 4 * (size_t)b;
    const int nx = (int)meta[0], ny = (int)meta[1];
    unsigned char* bp = a.bp + meta[2];
    const int K = a.K, ldc = K | 1;            // an odd row stride: a warp's double loads down a diagonal do not conflict
    double* C = meta[3] < 0 ? sm + 3 * (size_t)nx : a.cep + meta[3];
    const double* cx = C;
    const double* cy = C + (size_t)nx * ldc;

    // phase 1: the cepstra of X[b, :nx] (rows 0 .. nx-1 of C) and Y[b, :ny] (rows nx .. nx+ny-1)
    const double ln10_20 = 0.11512925464970229;          // ln(10) / 20
    for (int idx = tid; idx < (nx + ny) * K; idx += MCD_THREADS) {
        const int f = idx / K, k = idx - f * K;
        const float* x = f < nx ? a.X + ((size_t)b * a.Tx + f) * a.n_mels : a.Y + ((size_t)b * a.Ty + (f - nx)) * a.n_mels;
        const double* dk = a.dct + (size_t)k * a.n_mels;
        double c = 0.0;
        for (int m = 0; m < a.n_mels; ++m)
            c += ln10_20 * (a.max_db * (double)__ldg(x + m) - a.max_db + a.ref_db) * __ldg(dk + m);
        C[(size_t)f * ldc + k] = c;
    }
    __syncthreads();

    // phase 2: the anti-diagonals
    const double cost_scale = 4.3429448190325175;        // 10 / ln(10)
    double* prev2 = sm;                                   // diagonal d - 2
    double* prev1 = sm + nx;                              // diagonal d - 1
    double* cur = sm + 2 * (size_t)nx;
    for (int d = 0; d <= nx + ny - 2; ++d) {
        const int lo = max(0, d - (ny - 1)), hi = min(d, nx - 1);
        unsigned char* bpd = bp + diag_start(d, nx, ny) - lo;
        for (int i = lo + tid; i <= hi; i += MCD_THREADS) {
            const int j = d - i;
            const double* p = cx + (size_t)i * ldc;
            const double* q = cy + (size_t)j * ldc;
            double s = 0.0;
            for (int k = 0; k < K; ++k) {
                const double t = p[k] - q[k];
                s += t * t;
            }
            double v = cost_scale * sqrt(2.0 * s);
            unsigned char code = 0;
            if (d > 0) {
                // the first valid predecessor in the order diagonal, advance X, advance Y; a later one only when smaller
                double best;
                if (i > 0 && j > 0) {
                    best = prev2[i - 1];
                    if (prev1[i - 1] < best) { best = prev1[i - 1]; code = 1; }
                    if (prev1[i] < best) { best = prev1[i]; code = 2; }
                } else if (i > 0) {
                    best = prev1[i - 1]; code = 1;
                } else {
                    best = prev1[i]; code = 2;
                }
                v += best;
            }
            cur[i] = v;
            bpd[i] = code;
        }
        __syncthreads();
        double* x = prev2; prev2 = prev1; prev1 = cur; cur = x;
    }

    // the walk back from the end; the path goes out end first and is reversed below
    int* path = a.path ? a.path + (size_t)b * 2 * (a.Tx + a.Ty - 1) : nullptr;
    if (tid == 0) {
        int i = nx - 1, j = ny - 1, P = 0;
        while (true) {
            if (path) { path[2 * P] = i; path[2 * P + 1] = j; }
            ++P;
            if (i == 0 && j == 0) break;
            const int d = i + j, lo = max(0, d - (ny - 1));
            const unsigned char code = bp[diag_start(d, nx, ny) + i - lo];
            i -= code != 2;
            j -= code != 1;
        }
        a.pairs[b] = P;
        a.mcd[b] = prev1[nx - 1] / (double)P;
    }
    if (!path) return;
    __syncthreads();
    const int P = a.pairs[b], L = a.Tx + a.Ty - 1;
    for (int k = tid; k < L; k += MCD_THREADS) {
        if (k < P / 2) {
            const int r = P - 1 - k;
            const int i0 = path[2 * k], j0 = path[2 * k + 1];
            path[2 * k] = path[2 * r]; path[2 * k + 1] = path[2 * r + 1];
            path[2 * r] = i0; path[2 * r + 1] = j0;
        } else if (k >= P) {
            path[2 * k] = -1; path[2 * k + 1] = -1;
        }
    }
}

}  // namespace

void launch_mcd_dtw(const McdArgs& a, size_t smem, cudaStream_t s) {
    cudaError_t e = cudaFuncSetAttribute(mcd_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        mcd_dtw_kernel<<<a.B, MCD_THREADS, smem, s>>>(a);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) throw std::runtime_error(std::string("mcd_dtw_kernel launch failed: ") + cudaGetErrorString(e));
}

}  // namespace dctts
