// kernels_vocoder.cu -- Griffin-Lim vocoder (`spectrogram2wav`, reference utils.py:67-114) on the GPU.
// This is the first "next" row of SURVEY.md 8(f): the step right after the synthesis path, serial
// per-utterance CPU work in the reference (librosa), 51 inverse + 50 forward STFTs per utterance.
//
// One CTA of n_fft / 8 threads per STFT frame; the n_fft-point real transform is an n_fft/2-point complex Stockham FFT
// (radix-4 passes, plus one radix-2 pass where log2(n_fft/2) is odd; the first pass reads and the last pass writes
// registers, the others go through 2 x n_fft/2 x 8 B of shared memory), n_fft in {1024, 2048, 4096}.  The Hann window
// (win <= n_fft non-zero taps, centred in the frame) and librosa's conventions (center=True reflect padding, division by
// the summed squared window, n_fft/2 trimmed at both ends) are applied on the fly, so per Griffin-Lim iteration only the
// (B, T, 1 + n_fft/2) complex spectrum, the windowed frames and the waveform touch HBM:
//   voc_istft_kernel   spectrum row -> Hermitian extension -> IFFT -> x window -> frame buffer
//   voc_ola_kernel     overlap-add of the <= 5 frames covering a sample, / window sum-square
//   voc_stft_phase_kernel  reflect-padded frame x window -> FFT -> X = S * est / max(1e-8, |est|) (or the fast
//                          Griffin-Lim update, and the frame's spectral-convergence partial)
// plus de-normalisation (power law), the de-pre-emphasis IIR (float64 like scipy.signal.lfilter)
// and the frame energies librosa.effects.trim thresholds.
#include "kernels.cuh"
#include "numerics.cuh"

#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

namespace dctts {

// N = n_fft; the complex FFT has N / 2 points (real-input packing) and a CTA N / 8 threads, four values each
template <int N> struct VcSize {
    static constexpr int H = N / 2;
    static constexpr int THREADS = N / 8;
    static constexpr int LOG2H = N == 1024 ? 9 : N == 2048 ? 10 : 11;
    static constexpr int R4_SMEM = (LOG2H - 1) / 2;     // radix-4 passes that end in shared memory
    // __launch_bounds__ minimum of voc_istft_kernel: at 512 threads ptxas otherwise caps it at 32 registers and spills;
    // 0 (no minimum) leaves the smaller sizes as they were
    static constexpr int ISTFT_MIN_BLOCKS = N == 4096 ? 1 : 0;
    static_assert(N == 1024 || N == 2048 || N == 4096, "n_fft must be 1024, 2048 or 4096");
};

// Frames of utterance b: lengths[b] in a ragged call (clamped to [2, T]; the host checks the range), else T
__device__ __forceinline__ int voc_frames_of(const int* __restrict__ lengths, int b, int T) {
    return lengths ? min(max(__ldg(lengths + b), 2), T) : T;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// Index into [0, len) of sample u of np.pad(y, p, mode='reflect') at any pad length p (u < 0 lies in the left pad,
// u >= len in the right one).  A pad longer than the signal is reflected again and again, so the padded signal is
// periodic with period 2 (len - 1); numpy repeats the single sample of a signal of length 1.
__device__ __forceinline__ int reflect_index(int u, int len) {
    if (len == 1) return 0;
    const int period = 2 * (len - 1);
    if (u < 0) u = -u;
    if (u >= len) {
        u %= period;
        if (u >= len) u = period - u;
    }
    return u;
}

// N/2-point complex FFT, Stockham autosort, N/8 threads, one radix-4 butterfly per thread per pass.
// Entry: v[k] = x[tid + N/8 k]; exit: v[k] = X[tid + N/8 k] (natural order, no scaling).  The first pass reads
// registers; every radix-4 pass but a last one of length 4 writes one of the two ping-pong buffers s0 / s1 (one
// __syncthreads each, s0 first).  When log2(N/2) is even the last radix-4 pass (length 4, unit twiddles) stays in
// registers; when it is odd a radix-2 pass (length 2) does, on the pairs (v[0], v[2]) and (v[1], v[3]).
// tw[k] = exp(-2 pi i k / N), k < N.  Returns the buffer that no thread reads after the last barrier (free for the
// caller at once).
template <int N, bool INV>
__device__ __forceinline__ float2* fft_half(float2 (&v)[4], float2* s0, float2* s1, const float2* __restrict__ tw) {
    constexpr int T = VcSize<N>::THREADS, LOG2H = VcSize<N>::LOG2H;
    constexpr int LS_LAST = (LOG2H & 1) ? LOG2H - 3 : LOG2H - 2;      // ls of the last radix-4 pass
    const int tid = threadIdx.x;
    float2* buf = s0;
#pragma unroll
    for (int ls = 0; ls <= LS_LAST; ls += 2) {
        const int str = 1 << ls, q = tid & (str - 1), p = tid >> ls;
        const float2 a = v[0], b = v[1], c = v[2], d = v[3];
        const float2 apc = make_float2(a.x + c.x, a.y + c.y), amc = make_float2(a.x - c.x, a.y - c.y);
        const float2 bpd = make_float2(b.x + d.x, b.y + d.y), bmd = make_float2(b.x - d.x, b.y - d.y);
        const float2 jb = INV ? make_float2(bmd.y, -bmd.x) : make_float2(-bmd.y, bmd.x);      // (+-i)(b - d), sign folded: y1 = amc - jb
        float2 y0 = make_float2(apc.x + bpd.x, apc.y + bpd.y);
        float2 y1 = make_float2(amc.x - jb.x, amc.y - jb.y);
        float2 y2 = make_float2(apc.x - bpd.x, apc.y - bpd.y);
        float2 y3 = make_float2(amc.x + jb.x, amc.y + jb.y);
        if (!(LOG2H & 1) && ls == LS_LAST) { v[0] = y0; v[1] = y1; v[2] = y2; v[3] = y3; break; }   // n = 4: p = 0, unit twiddles
        const int i1 = 2 * (tid - q);
        float2 w1 = tw[i1], w2 = tw[2 * i1], w3 = tw[3 * i1];
        if (INV) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
        y1 = cmul(y1, w1); y2 = cmul(y2, w2); y3 = cmul(y3, w3);
        float2* o = buf + q + str * 4 * p;
        if (ls == 0) {
            reinterpret_cast<float4*>(o)[0] = make_float4(y0.x, y0.y, y1.x, y1.y);
            reinterpret_cast<float4*>(o)[1] = make_float4(y2.x, y2.y, y3.x, y3.y);
        } else { o[0] = y0; o[str] = y1; o[2 * str] = y2; o[3 * str] = y3; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = buf[tid + T * k];
        buf = (buf == s0) ? s1 : s0;
    }
    if (LOG2H & 1) {                                                                             // n = 2: unit twiddles
        const float2 a = v[0], b = v[1], c = v[2], d = v[3];
        v[0] = make_float2(a.x + c.x, a.y + c.y); v[2] = make_float2(a.x - c.x, a.y - c.y);
        v[1] = make_float2(b.x + d.x, b.y + d.y); v[3] = make_float2(b.x - d.x, b.y - d.y);
    }
    return (VcSize<N>::R4_SMEM & 1) ? s1 : s0;     // the buffer of the second-to-last shared-memory pass
}

template <int N>
__global__ void voc_twiddle_kernel(float2* tw) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < N) {
        double s, c;
        sincospi(-2.0 * (double)k / (double)N, &s, &c);
        tw[k] = make_float2((float)c, (float)s);
    }
}

// utils.py:78-85: amplitude target S = (10 ^ ((clip(z,0,1)*max_db - max_db + ref_db) * 0.05)) ^ power; X <- S (zero phase)
// STREAM (a streaming step, new_lo set): i runs over mag (B, n_new, F), whose row j of utterance b is frame new_lo[b] + j;
// the frames at or past lengths[b] are left alone.  Every vocoder kernel with a STREAM parameter compiles its STREAM = false
// instantiation, which the whole-signal calls launch, to the code it had before the streaming bounds existed.
template <bool STREAM>
__global__ void voc_prepare_kernel(const float* __restrict__ mag, float* __restrict__ S, float2* __restrict__ X, long long n,
                                   float max_db, float ref_db, float power, const int* __restrict__ lengths, int T, int F,
                                   const int* __restrict__ new_lo, int n_new) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    long long o = i;                                     // the element of S and X
    if constexpr (STREAM) {
        const long long row = i / F;
        const int b = (int)(row / n_new), t = __ldg(new_lo + b) + (int)(row % n_new);
        if (t >= min(__ldg(lengths + b), T)) return;
        o = ((long long)b * T + t) * F + i % F;
    } else if (lengths) {                                // rows past the utterance's frames: not read, zero
        const long long row = i / F;
        if ((int)(row % T) >= voc_frames_of(lengths, (int)(row / T), T)) { S[i] = 0.f; X[i] = make_float2(0.f, 0.f); return; }
    }
    float m = fminf(fmaxf(mag[i], 0.f), 1.f) * max_db - max_db + ref_db;
    float v = powf(powf(10.0f, m * 0.05f), power);
    S[o] = v;
    X[o] = make_float2(v, 0.f);
}

// librosa.core.istft, one frame: grid (T, B).  fr: (B, T, win) windowed time-domain frames.
// The N-point Hermitian inverse is an N/2-point complex one: with E/O the spectra of the even/odd
// samples, X[k] = E[k] + W^k O[k], X[k+N/2] = conj(X[N/2-k]) = E[k] - W^k O[k]; z = IFFT(E + i O)
// carries x[2n] in its real and x[2n+1] in its imaginary part.
// STREAM: frames frame_lo[b] + blockIdx.x.
template <int N, bool STREAM>
__global__ void __launch_bounds__(VcSize<N>::THREADS, VcSize<N>::ISTFT_MIN_BLOCKS)
voc_istft_kernel(const float2* __restrict__ X, float* __restrict__ fr, const float2* __restrict__ tw, const float* __restrict__ window,
                 int T, int F, int win, int lpad, const int* __restrict__ lengths, const int* __restrict__ frame_lo) {
    constexpr int H = VcSize<N>::H, NT = VcSize<N>::THREADS;
    __shared__ __align__(16) float2 s0[H];
    __shared__ __align__(16) float2 s1[H];
    const int b = blockIdx.y, tid = threadIdx.x;
    int t = blockIdx.x;
    if constexpr (STREAM) t += __ldg(frame_lo + b);
    if (t >= voc_frames_of(lengths, b, T)) return;       // whole CTA
    const float2* x = X + ((size_t)b * T + t) * F;
    float2 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kk = tid + NT * k;
        float2 xk = x[kk], xc = x[H - kk];
        if (kk == 0) { xk.y = 0.f; xc.y = 0.f; }        // ifft(...).real drops the imaginary parts of bins 0 and n_fft/2
        xc.y = -xc.y;
        const float2 e = make_float2(xk.x + xc.x, xk.y + xc.y), d = make_float2(xk.x - xc.x, xk.y - xc.y);
        float2 w = tw[kk]; w.y = -w.y;
        const float2 o = cmul(d, w);
        v[k] = make_float2(e.x - o.y, e.y + o.x);        // E + i O (the halves are folded into the 1/N below)
    }
    fft_half<N, true>(v, s0, s1, tw);
    float* o = fr + ((size_t)b * T + t) * win;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int m = 2 * (tid + NT * k) - lpad;         // frame sample 2n -> position in the window
        if (m >= 0 && m < win) o[m] = v[k].x * (1.0f / N) * window[m];
        if (m + 1 >= 0 && m + 1 < win) o[m + 1] = v[k].y * (1.0f / N) * window[m + 1];
    }
}

// overlap-add + window sum-square normalisation + centre trim: y (B, Ly), Ly = hop*(T-1).  Ragged call: utterance b has
// Tb frames and Ly_b = hop*(Tb-1) samples, the rest of its row is 0.  The table wss (T frames) equals the sum-square of Tb
// frames below Tb*hop + lpad (the later frames add zeros of the squared window there, which is exact); above it the
// sum is formed here from wsq, over frames < Tb in ascending order in float32 like voc_make_tables.
// STREAM: samples sample_lo[b] + blockIdx.x * blockDim.x + threadIdx.x.
template <int N, bool STREAM>
__global__ void voc_ola_kernel(const float* __restrict__ fr, const float* __restrict__ wss, float* __restrict__ y,
                               int T, int win, int lpad, int hop, int Ly, float tiny, const int* __restrict__ lengths,
                               const float* __restrict__ wsq, const int* __restrict__ sample_lo) {
    const int b = blockIdx.y;
    int sidx = blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (STREAM) sidx += __ldg(sample_lo + b);
    if (sidx >= Ly) return;
    const int Tb = voc_frames_of(lengths, b, T);
    if (sidx >= hop * (Tb - 1)) { y[(size_t)b * Ly + sidx] = 0.f; return; }
    const int u = sidx + N / 2;                          // index in the un-trimmed signal
    // frames t with lpad <= u - hop*t < lpad + win, in ascending order like librosa's loop
    int t_hi = (u - lpad) / hop;
    int t_lo = (u - lpad - win) / hop + 1;
    if (u - lpad - win < 0) t_lo = 0;
    t_hi = min(t_hi, Tb - 1);
    float acc = 0.f;
    for (int t = max(t_lo, 0); t <= t_hi; ++t) acc += fr[((size_t)b * T + t) * win + (u - hop * t - lpad)];
    float w;
    if (Tb == T || u < Tb * hop + lpad) {
        w = wss[u];
    } else {
        w = 0.f;
        for (int t = max(0, (u - N) / hop); t < Tb; ++t) {
            const int n = u - t * hop;
            if (n >= 0 && n < N) w += wsq[n];
        }
    }
    y[(size_t)b * Ly + sidx] = (w > tiny) ? acc / w : acc;
}

// librosa.core.stft of the current estimate, one frame, fused with the Griffin-Lim phase update
// (utils.py:101-104): X = S * est / max(1e-8, |est|).  grid (T, B).  Real input packed as
// z[n] = x[2n] + i x[2n+1]; est[k] = (Z[k] + conj Z[N/2-k]) / 2 - i W^k (Z[k] - conj Z[N/2-k]) / 2.
// MOM (fast Griffin-Lim): E (B, T, F) holds the previous iteration's raw estimate; the thread of bin k reads E[k], writes
// est[k] over it and updates with c = est - alpha E[k] (a float32 product, then a float32 difference, as numpy forms it for
// complex64): X = S * c / max(1e-8, |c|).  CONV: the frame's sum_k (S - |est|)^2 goes to part[b * T + t], summed in a fixed
// order (each thread's bins in ascending order, a warp butterfly, then the warp sums in ascending order; no atomics).
// STREAM: frames frame_lo[b] + blockIdx.x.
template <int N, bool MOM, bool CONV, bool STREAM>
__global__ void __launch_bounds__(VcSize<N>::THREADS) voc_stft_phase_kernel(const float* __restrict__ y, const float* __restrict__ S,
                                                                           float2* __restrict__ X, const float2* __restrict__ tw,
                                                                           const float* __restrict__ window, int T, int F, int win,
                                                                           int lpad, int hop, int Ly, const int* __restrict__ lengths,
                                                                           float2* __restrict__ E, float alpha, float* __restrict__ part,
                                                                           const int* __restrict__ frame_lo) {
    constexpr int H = VcSize<N>::H, NT = VcSize<N>::THREADS;
    __shared__ __align__(16) float2 s0[H];
    __shared__ __align__(16) float2 s1[H];
    int t = blockIdx.x;
    const int b = blockIdx.y, tid = threadIdx.x;
    if constexpr (STREAM) t += __ldg(frame_lo + b);
    const int Tb = voc_frames_of(lengths, b, T), Lyb = hop * (Tb - 1);
    if (t >= Tb) return;                                            // whole CTA
    const float* yb = y + (size_t)b * Ly;
    auto sample = [&](int n) -> float {
        const int m = n - lpad;
        if (m < 0 || m >= win) return 0.f;
        const int u = reflect_index(t * hop + n - N / 2, Lyb);     // np.pad(y, n_fft//2, mode='reflect')
        return yb[u] * window[m];
    };
    float2 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int n = 2 * (tid + NT * k); v[k] = make_float2(sample(n), sample(n + 1)); }
    float2* eb = MOM ? E + ((size_t)b * T + t) * F : nullptr;
    // MOM / CONV: this thread's S and previous estimates (index 4: bin n_fft/2, thread 0) are fetched before the FFT, so
    // that their latency hides behind it
    float sv[5] = {};
    float2 pv[5] = {};
    if constexpr (MOM || CONV) {
        const float* Sp = S + ((size_t)b * T + t) * F;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            sv[k] = Sp[tid + NT * k];
            if constexpr (MOM) pv[k] = eb[tid + NT * k];
        }
        if (tid == 0) {
            sv[4] = Sp[H];
            if constexpr (MOM) pv[4] = eb[H];
        }
    }
    float2* z = fft_half<N, false>(v, s0, s1, tw);                  // z was last read before the final barrier of the FFT
#pragma unroll
    for (int k = 0; k < 4; ++k) z[tid + NT * k] = v[k];
    __syncthreads();
    const float* Sb = S + ((size_t)b * T + t) * F;
    float2* x = X + ((size_t)b * T + t) * F;
    float dev = 0.f;                                                // CONV: this thread's sum of (S - |est|)^2
    auto emit = [&](int kk, float2 e, int slot) {
        if constexpr (MOM || CONV) {
            const float a = sv[slot];
            if constexpr (CONV) { const float d = a - sqrtf(e.x * e.x + e.y * e.y); dev = fmaf(d, d, dev); }
            if constexpr (MOM) {
                const float2 p = pv[slot];
                eb[kk] = e;
                e = make_float2(__fsub_rn(e.x, __fmul_rn(alpha, p.x)), __fsub_rn(e.y, __fmul_rn(alpha, p.y)));
            }
            const float mag = fmaxf(1e-8f, sqrtf(e.x * e.x + e.y * e.y));
            x[kk] = make_float2(a * (e.x / mag), a * (e.y / mag));
        } else {
            const float mag = fmaxf(1e-8f, sqrtf(e.x * e.x + e.y * e.y));
            const float a = Sb[kk];
            x[kk] = make_float2(a * (e.x / mag), a * (e.y / mag));
        }
    };
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kk = tid + NT * k;
        const float2 zk = v[k];
        float2 zc = z[(H - kk) & (H - 1)]; zc.y = -zc.y;
        const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
        const float2 d = make_float2(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
        const float2 o = cmul(make_float2(d.y, -d.x), tw[kk]);     // -i d W^k
        emit(kk, make_float2(e.x + o.x, e.y + o.y), k);
        if (kk == 0) emit(H, make_float2(zk.x - zk.y, 0.f), 4);    // bin n_fft/2: E[0] - O[0]
    }
    if constexpr (CONV) {
        dev = warp_sum(dev);
        float* red = reinterpret_cast<float*>(z == s0 ? s1 : s0);  // last read inside the FFT, before the barrier above
        if ((tid & 31) == 0) red[tid >> 5] = dev;
        __syncthreads();
        if (tid == 0) {
            float sum = 0.f;
            for (int w = 0; w < NT / 32; ++w) sum += red[w];
            part[(size_t)b * T + t] = sum;
        }
    }
}

// Spectral convergence ||S - |est_i||| / ||S|| of utterance b for i < n_hist: conv (B, n_hist) float64.  part (n_hist, B, T)
// holds the per-frame sums of voc_stft_phase_kernel<N, *, true, false>; frames t < T_b are summed in ascending order in float64.
// sum S^2 over the utterance's rows is formed once, in float64, each thread over a fixed stride, then a fixed tree.
// grid B, 256 threads.
__global__ void __launch_bounds__(256) voc_convergence_kernel(const float* __restrict__ S, const float* __restrict__ part,
                                                              double* __restrict__ conv, int B, int T, int F, int n_hist,
                                                              const int* __restrict__ lengths) {
    __shared__ double red[256];
    const int b = blockIdx.x, tid = threadIdx.x, Tb = voc_frames_of(lengths, b, T);
    const float* Sb = S + (size_t)b * T * F;
    double acc = 0.0;
    for (long long i = tid; i < (long long)Tb * F; i += 256) { const double v = Sb[i]; acc += v * v; }
    red[tid] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) red[tid] += red[tid + o];
        __syncthreads();
    }
    const double norm = sqrt(red[0]);
    for (int i = tid; i < n_hist; i += 256) {
        const float* p = part + ((size_t)i * B + b) * T;
        double num = 0.0;
        for (int t = 0; t < Tb; ++t) num += (double)p[t];
        conv[(size_t)b * n_hist + i] = sqrt(num) / norm;
    }
}

// scipy.signal.lfilter([1], [1, -c], wav): y[n] = x[n] + c*y[n-1], evaluated in float64 like scipy.
// The recurrence is linear, so it is cut into chunks of DE_LC samples: (1) every chunk's end state from a zero
// start, (2) per utterance the true state entering each chunk, carry[j] = end[j-1] + c^DE_LC * carry[j-1]
// (449 steps instead of 230 000), (3) every chunk again, seeded with its carry, writing float32.  Given the
// carry, step (3) is the reference's own sequence of float64 operations; the carries differ from the serial
// evaluation by float64 rounding only.  (One thread per utterance walking all samples took 5-13 ms.)
constexpr int DE_LC = 512;

// Ragged call: utterance b's chunks cover its Ly_b = hop (T_b - 1) samples only.
__device__ __forceinline__ int voc_samples_of(const int* __restrict__ lengths, int b, int T, int hop) {
    return hop * (voc_frames_of(lengths, b, T) - 1);
}

// A streaming de-emphasis's samples of row b: (first, count) from span[b] = [first, end)
__device__ __forceinline__ int2 voc_deemph_range(const int2* __restrict__ span, int b) {
    const int2 s = span[b];
    return make_int2(s.x, s.y - s.x);
}

// STREAM: the span's samples (voc_deemph_range) instead of the utterance's
template <bool STREAM>
__global__ void voc_deemph_local_kernel(const float* __restrict__ y, double* __restrict__ ends, int Ly, int nch, double c,
                                        const int* __restrict__ lengths, int T, int hop, const int2* __restrict__ span) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    int first = 0, Lyb = lengths ? voc_samples_of(lengths, b, T, hop) : Ly;
    if constexpr (STREAM) { const int2 r = voc_deemph_range(span, b); first = r.x; Lyb = r.y; }
    if (j >= (Lyb + DE_LC - 1) / DE_LC) return;
    const float* p = y + (size_t)b * Ly + first + (size_t)j * DE_LC;
    const int n = min(DE_LC, Lyb - j * DE_LC);
    double acc = 0.0;
    for (int i = 0; i < n; ++i) acc = (double)p[i] + c * acc;
    ends[(size_t)b * nch + j] = acc;
}

// STREAM: the span's chunks, and the carry into the first chunk is state[b] instead of 0
template <bool STREAM>
__global__ void voc_deemph_carry_kernel(double* __restrict__ ends, int nch, int B, double c, const int* __restrict__ lengths, int T,
                                        int hop, const int2* __restrict__ span, const double* __restrict__ state) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double cl = 1.0;
    for (int i = 0; i < DE_LC; ++i) cl *= c;
    double* e = ends + (size_t)b * nch;
    double carry = 0.0;
    int nchb = lengths ? (voc_samples_of(lengths, b, T, hop) + DE_LC - 1) / DE_LC : nch;
    if constexpr (STREAM) { carry = state[b]; nchb = (voc_deemph_range(span, b).y + DE_LC - 1) / DE_LC; }
    for (int j = 0; j < nchb; ++j) { const double local = e[j]; e[j] = carry; carry = local + cl * carry; }
}

// STREAM: the span's samples of `in` (another buffer than y) into y, and the last chunk's thread stores the state after its
// last sample; else y in place.
template <bool STREAM>
__global__ void voc_deemph_apply_kernel(float* __restrict__ y, const double* __restrict__ carry, int Ly, int nch, double c,
                                        const int* __restrict__ lengths, int T, int hop, const int2* __restrict__ span,
                                        const float* __restrict__ in, double* __restrict__ state) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if constexpr (STREAM) {
        const int2 r = voc_deemph_range(span, b);
        const int Lyb = r.y;
        if (j >= (Lyb + DE_LC - 1) / DE_LC) return;
        const size_t o = (size_t)b * Ly + r.x + (size_t)j * DE_LC;
        float* p = y + o;
        const float* q = in + o;
        const int n = min(DE_LC, Lyb - j * DE_LC);
        double acc = carry[(size_t)b * nch + j];
        for (int i = 0; i < n; ++i) { acc = (double)q[i] + c * acc; p[i] = (float)acc; }
        if ((j + 1) * DE_LC >= Lyb) state[b] = acc;
    } else {
        const int Lyb = lengths ? voc_samples_of(lengths, b, T, hop) : Ly;
        if (j >= (Lyb + DE_LC - 1) / DE_LC) return;
        float* p = y + (size_t)b * Ly + (size_t)j * DE_LC;
        const int n = min(DE_LC, Lyb - j * DE_LC);
        double acc = carry[(size_t)b * nch + j];
        for (int i = 0; i < n; ++i) { acc = (double)p[i] + c * acc; p[i] = (float)acc; }
    }
}

// A waveform sample as float32: float input as is, int16 PCM as value / 32768 (exact: what utils._load_wav returns)
__device__ __forceinline__ float wav_sample(const float* __restrict__ y, long long i) { return y[i]; }
__device__ __forceinline__ float wav_sample(const int16_t* __restrict__ y, long long i) { return (float)y[i] * (1.0f / 32768.0f); }

// librosa.feature.rmse(y, flen, fhop)**2 of centred frame f (reflect padding) of the signal yb[0, Ly), Ly >= 2.  256
// threads; the result is valid in thread 0.
template <typename In>
__device__ __forceinline__ float frame_mse(const In* __restrict__ yb, int Ly, int f, int flen, int fhop, float* red) {
    float acc = 0.f;
    for (int n = threadIdx.x; n < flen; n += 256) {
        const float v = wav_sample(yb, reflect_index(f * fhop + n - flen / 2, Ly));
        acc = fmaf(v, v, acc);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0)
        for (int i = 0; i < 8; ++i) t += red[i];
    return t / (float)flen;
}

// frame energies of B equally long signals: mse (B, nfr), grid (nfr, B)
// (ragged call: utterance b's 1 + Ly_b / fhop frames over its Ly_b samples; the other CTAs of its row leave)
__global__ void __launch_bounds__(256) voc_frame_mse_kernel(const float* __restrict__ y, float* __restrict__ mse, int Ly, int nfr,
                                                           int flen, int fhop, const int* __restrict__ lengths, int T, int hop) {
    __shared__ float red[8];
    const int Lyb = lengths ? voc_samples_of(lengths, blockIdx.y, T, hop) : Ly;
    if ((int)blockIdx.x >= 1 + Lyb / fhop) return;                  // whole CTA
    const float m = frame_mse(y + (size_t)blockIdx.y * Ly, Lyb, blockIdx.x, flen, fhop, red);
    if (threadIdx.x == 0) mse[(size_t)blockIdx.y * nfr + blockIdx.x] = m;
}

// ---------------------------------------------------------------------------------------- features
// The utterance of flattened frame g: seg[b].f0 <= g < seg[b + 1].f0 (seg has B + 1 entries).
__device__ __forceinline__ int feat_segment(const FeatSeg* __restrict__ seg, int B, int g) {
    int lo = 0, hi = B;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (seg[mid].f0 <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// frame energies of B ragged signals for librosa.effects.trim (2048-sample frames, hop 512): one CTA per frame over the
// flattened batch, mse[g] for frame g - seg[b].f0 of utterance b
template <typename In>
__global__ void __launch_bounds__(256) feat_frame_mse_kernel(const In* __restrict__ wav, const FeatSeg* __restrict__ seg, int B,
                                                            float* __restrict__ mse) {
    __shared__ float red[8];
    const int g = blockIdx.x, b = feat_segment(seg, B, g);
    const FeatSeg sg = seg[b];
    const float m = frame_mse(wav + sg.src, sg.len, g - sg.f0, 2048, 512, red);
    if (threadIdx.x == 0) mse[g] = m;
}

// get_spectrograms (reference utils.py:20-65) for B trimmed utterances, one CTA per STFT frame over the flattened batch
// (seg: the utterance's trimmed start, length and first flattened frame): pre-emphasis (float32 multiply then subtract,
// like numpy), reflect-padded Hann frame, the same real-packed FFT, |X|, the mel filterbank (each mel bin is a
// contiguous run of FFT bins), 20 log10, normalisation.  Frame t of utterance b writes mag row b * mag_rows + t; frames
// with t % r == 0 also write mel row b * mel_rows + t / r (load_spectrograms' reduction, utils.py:155-160).
template <int N, typename In>
__global__ void __launch_bounds__(VcSize<N>::THREADS) feat_stft_mel_kernel(const In* __restrict__ wav, const FeatSeg* __restrict__ seg,
                                                                          int B, float preemph,
                                                                          float* __restrict__ mag_out, float* __restrict__ mel_out,
                                                                          int mag_rows, int mel_rows, int r,
                                                                          const float* __restrict__ melw, const int2* __restrict__ melrange,
                                                                          const float2* __restrict__ tw, const float* __restrict__ window,
                                                                          int F, int n_mels, int win, int lpad, int hop, float ref_db,
                                                                          float max_db) {
    constexpr int H = VcSize<N>::H, NT = VcSize<N>::THREADS;
    __shared__ __align__(16) float2 s0[H];
    __shared__ __align__(16) float2 s1[H];
    const int tid = threadIdx.x, b = feat_segment(seg, B, blockIdx.x);
    const FeatSeg sg = seg[b];
    const int t = blockIdx.x - sg.f0, len = sg.len;
    const In* y = wav + sg.src;
    auto sample = [&](int n) -> float {
        const int m = n - lpad;
        if (m < 0 || m >= win) return 0.f;
        const int u = reflect_index(t * hop + n - N / 2, len);     // np.pad(y, n_fft//2, mode='reflect')
        const float v = (u > 0) ? __fsub_rn(wav_sample(y, u), __fmul_rn(preemph, wav_sample(y, u - 1))) : wav_sample(y, 0);   // utils.py:39
        return v * window[m];
    };
    float2 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int n = 2 * (tid + NT * k); v[k] = make_float2(sample(n), sample(n + 1)); }
    float2* z = fft_half<N, false>(v, s0, s1, tw);
#pragma unroll
    for (int k = 0; k < 4; ++k) z[tid + NT * k] = v[k];
    __syncthreads();
    float* lin = reinterpret_cast<float*>(z == s0 ? s1 : s0);   // |X[k]|, k <= N/2 (the other buffer was last read inside the FFT)
    float* mo = mag_out + ((size_t)b * mag_rows + t) * F;
    auto emit = [&](int kk, float2 e) {
        const float a = sqrtf(e.x * e.x + e.y * e.y);
        lin[kk] = a;
        const float db = 20.0f * log10f(fmaxf(1e-5f, a));
        mo[kk] = fminf(fmaxf((db - ref_db + max_db) / max_db, 1e-8f), 1.0f);
    };
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kk = tid + NT * k;
        const float2 zk = v[k];
        float2 zc = z[(H - kk) & (H - 1)]; zc.y = -zc.y;
        const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
        const float2 d = make_float2(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
        const float2 o = cmul(make_float2(d.y, -d.x), tw[kk]);
        emit(kk, make_float2(e.x + o.x, e.y + o.y));
        if (kk == 0) emit(H, make_float2(zk.x - zk.y, 0.f));
    }
    if (t % r != 0) return;                                // a frame the reduction drops: mag only
    __syncthreads();
    float* mel_row = mel_out + ((size_t)b * mel_rows + t / r) * n_mels;
    const int warp = tid >> 5, lane = tid & 31;
    for (int m = warp; m < n_mels; m += NT / 32) {
        const int2 r = melrange[m];
        const float* w = melw + (size_t)m * F;
        float acc = 0.f;
        for (int k = r.x + lane; k < r.y; k += 32) acc = fmaf(w[k], lin[k], acc);
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            const float db = 20.0f * log10f(fmaxf(1e-5f, acc));
            mel_row[m] = fminf(fmaxf((db - ref_db + max_db) / max_db, 1e-8f), 1.0f);
        }
    }
}

// ---------------------------------------------------------------------------------------- host
bool voc_fft_size_ok(int n_fft) { return n_fft == 1024 || n_fft == 2048 || n_fft == 4096; }

// Calls f(std::integral_constant<int, n_fft>): the kernel instantiation for the handle's n_fft
template <typename Fn>
static void voc_dispatch(int n_fft, Fn&& f) {
    switch (n_fft) {
        case 1024: f(std::integral_constant<int, 1024>{}); break;
        case 2048: f(std::integral_constant<int, 2048>{}); break;
        case 4096: f(std::integral_constant<int, 4096>{}); break;
        default: throw std::runtime_error("vocoder: n_fft = " + std::to_string(n_fft) + " (supported: 1024, 2048, 4096)");
    }
}

void voc_make_tables(int n_fft, float2* tw_dev, float* window_dev, float* wss_dev, int T, int win, int hop, cudaStream_t s,
                     float* wsq_dev) {
    voc_dispatch(n_fft, [&](auto n) { voc_twiddle_kernel<decltype(n)::value><<<(n_fft + 255) / 256, 256, 0, s>>>(tw_dev); });
    // periodic Hann of win taps (scipy get_window('hann', win, fftbins=True)) and librosa's window_sumsquare,
    // accumulated in float32 in frame order like the reference
    std::vector<float> w(win);
    for (int n = 0; n < win; ++n) w[n] = (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * (double)n / (double)win));
    const int lpad = (n_fft - win) / 2;
    const int n_tot = n_fft + hop * (T - 1);
    std::vector<float> wss(n_tot, 0.f);
    std::vector<float> wsq(n_fft, 0.f);
    for (int n = 0; n < win; ++n) { const double d = 0.5 - 0.5 * std::cos(2.0 * M_PI * (double)n / (double)win); wsq[lpad + n] = (float)(d * d); }
    for (int t = 0; t < T; ++t)
        for (int n = 0; n < n_fft && t * hop + n < n_tot; ++n) wss[t * hop + n] += wsq[n];
    cudaMemcpyAsync(window_dev, w.data(), win * sizeof(float), cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(wss_dev, wss.data(), n_tot * sizeof(float), cudaMemcpyHostToDevice, s);
    if (wsq_dev) cudaMemcpyAsync(wsq_dev, wsq.data(), n_fft * sizeof(float), cudaMemcpyHostToDevice, s);
    cudaStreamSynchronize(s);
}

// librosa.filters.mel(sr, n_fft, n_mels): Slaney scale, fmin 0, fmax sr/2, area-normalised triangles (float64 here,
// float32 on the device); range[m] = [first, last+1) non-zero FFT bin of mel bin m.
void feat_make_mel_basis(int sr, int n_fft, int n_mels, std::vector<float>& w, std::vector<int>& range) {
    const int F = 1 + n_fft / 2;
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
    auto hz2mel = [&](double f) { return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp; };
    auto mel2hz = [&](double m) { return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m; };
    std::vector<double> mel_f(n_mels + 2);
    const double m_lo = hz2mel(0.0), m_hi = hz2mel(sr / 2.0);
    for (int i = 0; i < n_mels + 2; ++i) mel_f[i] = mel2hz(m_lo + (m_hi - m_lo) * (double)i / (double)(n_mels + 1));
    w.assign((size_t)n_mels * F, 0.f);
    range.assign(2 * (size_t)n_mels, 0);
    for (int i = 0; i < n_mels; ++i) {
        const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
        int first = -1, last = -1;
        for (int k = 0; k < F; ++k) {
            const double f = (sr / 2.0) * (double)k / (double)(F - 1);
            const double lower = (f - mel_f[i]) / (mel_f[i + 1] - mel_f[i]);
            const double upper = (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1]);
            const double v = std::max(0.0, std::min(lower, upper)) * enorm;
            w[(size_t)i * F + k] = (float)v;
            if (v > 0.0) { if (first < 0) first = k; last = k; }
        }
        range[2 * i] = first < 0 ? 0 : first;
        range[2 * i + 1] = first < 0 ? 0 : last + 1;
    }
}

void feat_frame_mse(const void* wav, int dtype, const FeatSeg* seg, int B, int frames, float* mse, cudaStream_t s) {
    if (dtype == 1)
        feat_frame_mse_kernel<int16_t><<<frames, 256, 0, s>>>(static_cast<const int16_t*>(wav), seg, B, mse);
    else
        feat_frame_mse_kernel<float><<<frames, 256, 0, s>>>(static_cast<const float*>(wav), seg, B, mse);
}

void feat_run(const FeatArgs& a, cudaStream_t s) {
    const int2* range = reinterpret_cast<const int2*>(a.melrange);
    voc_dispatch(2 * (a.F - 1), [&](auto n) {
        constexpr int N = decltype(n)::value;
        const int lpad = (N - a.win) / 2;
        if (a.dtype == 1)
            feat_stft_mel_kernel<N, int16_t><<<a.frames, VcSize<N>::THREADS, 0, s>>>(
                static_cast<const int16_t*>(a.wav), a.seg, a.B, a.preemph, a.mag, a.mel, a.mag_rows, a.mel_rows, a.r, a.melw, range,
                a.tw, a.window, a.F, a.n_mels, a.win, lpad, a.hop, a.ref_db, a.max_db);
        else
            feat_stft_mel_kernel<N, float><<<a.frames, VcSize<N>::THREADS, 0, s>>>(
                static_cast<const float*>(a.wav), a.seg, a.B, a.preemph, a.mag, a.mel, a.mag_rows, a.mel_rows, a.r, a.melw, range,
                a.tw, a.window, a.F, a.n_mels, a.win, lpad, a.hop, a.ref_db, a.max_db);
    });
}

// ---------------------------------------------------------------------------------------- resampling
// resampy 0.2 resample_f for output t of one utterance, one thread per output sample over the flattened batch.  Every
// float64 operation is an explicit round-to-nearest intrinsic, so nothing is contracted into an FMA (numba does not
// contract either).  `win` is the unscaled interp_win; for ratio < 1 resampy scales it by the ratio before taking
// interp_delta = diff(interp_win), and so does `tap`.  The accumulator is float32 and every tap rounds
// float32(double(y) + weight * double(x)), numba's semantics for `y[t] += weight * x[...]` with a float32 y.
template <typename In>
__global__ void __launch_bounds__(256) resample_kernel(const In* __restrict__ wav, const ResampleUtt* __restrict__ utt, int B,
                                                       const TimeSeg* __restrict__ seg, const double* __restrict__ win,
                                                       float* __restrict__ out, long long total) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    int lo = 0, hi = B;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (utt[mid].dst <= g) lo = mid; else hi = mid;
    }
    const ResampleUtt u = utt[lo];
    const long long t = g - u.dst;
    const In* x = wav + u.src;
    if (t >= u.n_valid) { out[g] = 0.f; return; }                        // librosa util.fix_length
    if (u.index_step == 0) { out[g] = wav_sample(x, t); return; }        // librosa: orig_sr == target_sr returns y
    int a = u.seg0, b = u.seg0 + u.nseg;
    while (b - a > 1) {
        const int mid = (a + b) >> 1;
        if (seg[mid].t0 <= t) a = mid; else b = mid;
    }
    const double reg = __dadd_rn(seg[a].v0, __dmul_rn((double)(t - seg[a].t0), seg[a].step));   // exact (see TimeSeg)
    const double ratio = u.ratio, scale = u.scale;
    const bool scaled = ratio < 1.0;
    const int step = u.index_step;
    double eta;
    auto weight = [&](int j) -> double {                  // interp_win[j] + eta * interp_delta[j]
        double w0 = win[j], d = 0.0;
        if (scaled) w0 = __dmul_rn(w0, ratio);
        if (j + 1 < RS_NWIN) {
            const double w1 = scaled ? __dmul_rn(win[j + 1], ratio) : win[j + 1];
            d = __dsub_rn(w1, w0);
        }
        return __dadd_rn(w0, __dmul_rn(eta, d));
    };
    const long long n = (long long)reg;
    double frac = __dmul_rn(scale, __dsub_rn(reg, (double)n));
    double index_frac = __dmul_rn(frac, (double)RS_TABLE);
    int offset = (int)index_frac;
    eta = __dsub_rn(index_frac, (double)offset);
    float y = 0.f;
    const long long i_max = min(n + 1, (long long)((RS_NWIN - offset) / step));          // left wing
    for (int i = 0; i < i_max; ++i)
        y = (float)__dadd_rn((double)y, __dmul_rn(weight(offset + i * step), (double)wav_sample(x, n - i)));
    frac = __dsub_rn(scale, frac);
    index_frac = __dmul_rn(frac, (double)RS_TABLE);
    offset = (int)index_frac;
    eta = __dsub_rn(index_frac, (double)offset);
    const long long k_max = min((long long)u.n_in - n - 1, (long long)((RS_NWIN - offset) / step));   // right wing
    for (int k = 0; k < k_max; ++k)
        y = (float)__dadd_rn((double)y, __dmul_rn(weight(offset + k * step), (double)wav_sample(x, n + k + 1)));
    out[g] = y;
}

namespace {
// I0 by its power series sum (x/2)^2k / (k!)^2, in long double
double bessel_i0(double x) {
    const long double q = (long double)x * x / 4;
    long double term = 1, sum = 1;
    for (int k = 1; k < 1000 && term > sum * 1e-22L; ++k) {
        term *= q / ((long double)k * k);
        sum += term;
    }
    return (double)sum;
}
}  // namespace

// resampy 0.2 filters.sinc_window(num_zeros=64, precision=9, window=kaiser(beta), rolloff) for 'kaiser_best':
// rolloff * sinc(rolloff * linspace(0, 64, 64*512 + 1)) times the right half of scipy.signal.kaiser(2*64*512 + 1, beta).
void resample_filter_table(std::vector<double>& win) {
    const double beta = 14.769656459379492, rolloff = 0.9475937167399596, pi = 3.141592653589793;
    const int n = RS_NWIN - 1;
    win.resize(RS_NWIN);
    const double i0_beta = bessel_i0(beta);
    for (int j = 0; j <= n; ++j) {
        const double z = rolloff * ((double)j * (64.0 / n));                 // linspace: j * step, exact here
        const double y = pi * (z == 0.0 ? 1.0e-20 : z);                      // np.sinc
        const double r = (double)j / n;                                      // (m - alpha) / alpha, m = n + j
        win[j] = bessel_i0(beta * std::sqrt(1.0 - r * r)) / i0_beta * (rolloff * (std::sin(y) / y));
    }
}

// The register values 0, inc, fl(inc + inc), ... of n_out outputs as affine segments.  Inside one binade
// [2^k, 2^(k+1)) every double is a multiple V g of g = 2^(k-52), and fl(V g + inc) = (V + S) g with S = inc / g rounded
// to the nearest integer, as long as the result stays below 2^(k+1): one segment per binade.  When inc / g lies exactly
// halfway, rounding goes to the even neighbour, so from an even V every step adds the even one of S0, S0 + 1; an odd V
// takes one explicit addition first.  The first value (0) and each addition that leaves a binade are done in float64.
// Appends to `out`; returns the number of segments.
int resample_time_register(long long n_out, double inc, std::vector<TimeSeg>& out) {
    const size_t first = out.size();
    long long t = 0;
    double v = 0.0;
    while (t < n_out) {
        long long S = -1, V = 0;
        double g = 0.0;
        if (v > 0.0) {
            int e;
            std::frexp(v, &e);                                  // v in [2^(e-1), 2^e)
            g = std::ldexp(1.0, e - 53);
            V = (long long)(v / g);                             // exact, in [2^52, 2^53)
            const double q = inc / g, q0 = std::floor(q), fr = q - q0;   // exact (v >= inc, so q < 2^53)
            const long long S0 = (long long)q0;
            if (fr > 0.5) S = S0 + 1;
            else if (fr < 0.5) S = S0;
            else if (!(V & 1)) S = S0 + (S0 & 1);
        }
        if (S < 0) {                                            // zero, or a tie from an odd V: one explicit addition
            out.push_back(TimeSeg{t, v, 0.0});
            ++t;
            v = v + inc;
            continue;
        }
        const long long H = 1ll << 53;
        const long long m = S > 0 ? (H - 1 - V) / S : n_out;    // additions that stay inside the binade
        const long long len = std::min(m + 1, n_out - t);
        out.push_back(TimeSeg{t, v, (double)S * g});
        t += len;
        v = (double)(V + (len - 1) * S) * g;
        if (t < n_out) v = v + inc;                             // the addition that leaves the binade
    }
    return (int)(out.size() - first);
}

void resample_run(const void* wav, int dtype, const ResampleUtt* utt, int B, const TimeSeg* seg, const double* win, float* out,
                  long long total, cudaStream_t s) {
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == 1)
        resample_kernel<int16_t><<<grid, 256, 0, s>>>(static_cast<const int16_t*>(wav), utt, B, seg, win, out, total);
    else
        resample_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(wav), utt, B, seg, win, out, total);
}

int voc_launches_per_call(int n_iter, bool convergence) { return 1 + 3 * n_iter + 2 + 3 + 1 + (convergence ? 2 : 0); }
size_t voc_deemph_scratch_bytes(int B, int T, int hop) { return (size_t)B * ((hop * (T - 1) + DE_LC - 1) / DE_LC) * sizeof(double); }

// The stages of voc_run, each a fixed sequence of launches (dctts_vocoder_stage runs them one at a time).
void voc_prepare(const VocoderArgs& a, cudaStream_t s) {
    const long long n = (long long)a.B * (a.new_lo ? a.n_new : a.T) * a.F;
    auto kern = a.new_lo ? voc_prepare_kernel<true> : voc_prepare_kernel<false>;
    kern<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a.mag, a.S, a.X, n, a.max_db, a.ref_db, a.power, a.lengths, a.T, a.F, a.new_lo,
                                                     a.n_new);
}

void voc_istft(const VocoderArgs& a, cudaStream_t s) {
    voc_dispatch(2 * (a.F - 1), [&](auto n) {
        constexpr int N = decltype(n)::value;
        const int Ly = a.hop * (a.T - 1), lpad = (N - a.win) / 2;
        const bool st = a.frame_lo != nullptr;           // a streaming step sets frame_lo and sample_lo together
        const int nt = st ? a.n_active : a.T, ns = st ? a.n_samples : Ly;
        auto istft = st ? voc_istft_kernel<N, true> : voc_istft_kernel<N, false>;
        auto ola = st ? voc_ola_kernel<N, true> : voc_ola_kernel<N, false>;
        istft<<<dim3(nt, a.B), VcSize<N>::THREADS, 0, s>>>(a.X, a.frames, a.tw, a.window, a.T, a.F, a.win, lpad, a.lengths, a.frame_lo);
        ola<<<dim3((ns + 255) / 256, a.B), 256, 0, s>>>(a.frames, a.wss, a.wav, a.T, a.win, lpad, a.hop, Ly, 1.17549435e-38f,
                                                       a.lengths, a.wsq, a.sample_lo);
    });
}

void voc_stft_phase(const VocoderArgs& a, cudaStream_t s, int it) {
    float* part = a.part ? a.part + (size_t)it * a.B * a.T : nullptr;
    voc_dispatch(2 * (a.F - 1), [&](auto n) {
        constexpr int N = decltype(n)::value;
        const int Ly = a.hop * (a.T - 1), lpad = (N - a.win) / 2;
        auto launch = [&](auto kern) {
            kern<<<dim3(a.frame_lo ? a.n_active : a.T, a.B), VcSize<N>::THREADS, 0, s>>>(
                a.wav, a.S, a.X, a.tw, a.window, a.T, a.F, a.win, lpad, a.hop, Ly, a.lengths, a.E, a.alpha, part, a.frame_lo);
        };
        if (a.frame_lo) {                              // a streaming step keeps no convergence history
            if (a.E) launch(voc_stft_phase_kernel<N, true, false, true>); else launch(voc_stft_phase_kernel<N, false, false, true>);
        } else if (a.E) {
            if (part) launch(voc_stft_phase_kernel<N, true, true, false>); else launch(voc_stft_phase_kernel<N, true, false, false>);
        } else {
            if (part) launch(voc_stft_phase_kernel<N, false, true, false>); else launch(voc_stft_phase_kernel<N, false, false, false>);
        }
    });
}

void voc_convergence(const VocoderArgs& a, cudaStream_t s) {
    voc_convergence_kernel<<<a.B, 256, 0, s>>>(a.S, a.part, a.conv, a.B, a.T, a.F, a.n_iter + 1, a.lengths);
}

void voc_deemph(const VocoderArgs& a, cudaStream_t s) {
    const int Ly = a.hop * (a.T - 1), nch = ((a.span ? a.n_span : Ly) + DE_LC - 1) / DE_LC;
    const dim3 gch((nch + 63) / 64, a.B);
    const bool st = a.span != nullptr;                   // a streaming step sets span, deemph_in and state together
    auto local = st ? voc_deemph_local_kernel<true> : voc_deemph_local_kernel<false>;
    auto carry = st ? voc_deemph_carry_kernel<true> : voc_deemph_carry_kernel<false>;
    auto apply = st ? voc_deemph_apply_kernel<true> : voc_deemph_apply_kernel<false>;
    local<<<gch, 64, 0, s>>>(st ? a.deemph_in : a.wav, a.deemph, Ly, nch, a.preemphasis, a.lengths, a.T, a.hop, a.span);
    carry<<<(a.B + 31) / 32, 32, 0, s>>>(a.deemph, nch, a.B, a.preemphasis, a.lengths, a.T, a.hop, a.span, a.state);
    apply<<<gch, 64, 0, s>>>(a.wav, a.deemph, Ly, nch, a.preemphasis, a.lengths, a.T, a.hop, a.span, a.deemph_in, a.state);
}

void voc_energies(const VocoderArgs& a, cudaStream_t s) {
    const int Ly = a.hop * (a.T - 1), nfr = 1 + Ly / 512;
    voc_frame_mse_kernel<<<dim3(nfr, a.B), 256, 0, s>>>(a.wav, a.mse, Ly, nfr, 2048, 512, a.lengths, a.T, a.hop);
}

void voc_run(const VocoderArgs& a, cudaStream_t s) {
    voc_prepare(a, s);
    for (int it = 0; it <= a.n_iter; ++it) {
        voc_istft(a, s);
        if (it < a.n_iter) voc_stft_phase(a, s, it);
    }
    if (a.part) {                       // est_{n_iter}: one more STFT of the final waveform (X is free now, E is not needed)
        VocoderArgs f = a;
        f.E = nullptr;
        voc_stft_phase(f, s, a.n_iter);
        voc_convergence(a, s);
    }
    voc_deemph(a, s);
    voc_energies(a, s);
}

}  // namespace dctts
