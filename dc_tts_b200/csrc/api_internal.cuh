// api_internal.cuh -- what the host library's translation units share: the handle and its buffers, the error macros,
// the C-ABI guard, and the few functions one stage calls in another (DESIGN.md section 1).  Not installed.
#pragma once
#include "../../include/dctts.h"
#include "kernels.cuh"
#include "kernels_tc.cuh"
#include "kernels_decode.cuh"

#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <thread>
#include <vector>

using namespace dctts;

#define CUDA_CHECK(expr)                                                                     \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            char _buf[512];                                                                  \
            snprintf(_buf, sizeof(_buf), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                     __FILE__, __LINE__);                                                    \
            throw std::runtime_error(_buf);                                                  \
        }                                                                                    \
    } while (0)

#define REQUIRE(cond, msg)                                   \
    do {                                                     \
        if (!(cond)) throw std::runtime_error(std::string(msg)); \
    } while (0)

namespace dctts::api {

extern std::string g_create_error;   // why the last dctts_create failed, or the last call on a null handle

inline int roundup(int x, int m) { return (x + m - 1) / m * m; }

enum Kind { K_C = 0, K_HC = 1, K_D = 2 };

struct LayerDev {
    std::string scope;   // full scope, e.g. "SSRN/HC_5"
    int kind = K_C;
    int cin = 0, cout = 0, size = 1, rate = 1;
    bool causal = false;
    int act = 0;
    int nconv = 0, ldw = 0;
    float* W = nullptr;      // [size][cin][ldw]
    float* bias = nullptr;   // [ldw]
    float *g1 = nullptr, *b1 = nullptr, *g2 = nullptr, *b2 = nullptr;
    // tensor-core path: split-fp16 K-major weight planes [ncta*bn][ntaps*cin_pad], pre-scaled
    struct TcPack {
        bool ok = false;
        int mode = 0, ntaps = 0, kb_per_tap = 0, Ktot = 0, ncta = 1, bn = 0, half = 0, nrows = 0;
        float inv_scale = 1.f;
        __half *Whi = nullptr, *Wlo = nullptr;
        CUtensorMap mWhi, mWlo;
    } tc;
};

struct HostParam {
    std::vector<float> data;
    std::vector<int64_t> shape;
};

// A device allocation that grows on demand and is freed with its owner; move-only.
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), bytes(std::exchange(o.bytes, 0)) {}
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(bytes, o.bytes); return *this; }
    ~DevBuf() { if (p) cudaFree(p); }
    // At least n bytes; the contents are not kept.  A growth first waits for all work on the device, since kernels queued
    // on any stream may still read the old allocation; so no growth may happen inside a stream capture.
    void ensure(size_t n) {
        if (n <= bytes) return;
        if (p) { CUDA_CHECK(cudaDeviceSynchronize()); CUDA_CHECK(cudaFree(p)); }
        p = nullptr; bytes = 0;
        CUDA_CHECK(cudaMalloc(&p, n));
        bytes = n;
    }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

}  // namespace dctts::api

using namespace dctts::api;

struct dctts_handle_s {
    dctts_hparams hp{};
    int device = 0;
    int num_sms = 132;            // streaming multiprocessors of the device (set at creation)
    int F = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;      // device->host copies of finished spectrogram chunks (dctts_synthesize_host)
    cudaEvent_t chunk_done[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    std::string err;

    std::map<std::string, HostParam> staged;
    bool committed = false;
    int64_t n_params = 0;

    std::vector<LayerDev> textenc, audioenc, audiodec, ssrn;
    std::map<std::string, LayerDev*> by_scope;
    std::map<std::string, float*> dev_vec;    // every committed variable (flat copy) by TF name
    std::deque<DevBuf> param_bufs;            // every committed parameter plane; a deque keeps the pointers that tensor maps and DecParams hold
    float* embed_table = nullptr;
    DevBuf pack_max;              // weight packing (kernels_pack.cu): every layer's max |W| (float bits)
    // the variables changed since the planes and the decode stream were packed (mark_synthesis_stale): synthesis runs on
    // the fp32 kernels with the graph-per-frame decode until dctts_refresh_synthesis packs them again
    bool synth_stale = false;

    // workspace (sized for ws_B utterances)
    int ws_B = 0;
    DevBuf scratch, act0, act1;
    DevBuf tickets;               // arrival counters of the fused GEMM + LN launches (2 ints per 16-row block)
    DevBuf kv;                    // (B, N, 2d) TextEnc output
    DevBuf ybuf;                  // (B, T, n_mels) generated mels
    DevBuf rbuf;                  // (B, T, 2d)
    std::vector<DevBuf> ae_out;   // AudioEnc per-layer outputs (B, T, d)
    std::vector<DevBuf> ad_out;   // AudioDec per-layer outputs (B, T, d | n_mels)
    DevBuf ad_sig;                // scratch for sigmoid(logits) in full-graph mode
    DevBuf ibuf;                  // ints: j, p_cur[B], p_next[B], p_prev[B], p_hist[B*T]
    DevBuf pathbuf;               // ints of a decode along a window path: lengths[B], path[B*T], argmax[B*T]
    void* path_pinned = nullptr;  // pinned staging of the host arrays upload_host copies to the device (api_synth.cu),
    size_t path_pinned_bytes = 0; // reused once path_uploaded has fired
    cudaEvent_t path_uploaded = nullptr;
    // the aligner (dctts_align_search, dctts_text2mel_align): back-pointers (B, T, N) uint8, lengths and ends (2B) ints, and
    // the alignments (B, max_N, T) when the caller does not ask for them
    struct { DevBuf bp, meta, A; } align;
    // MCD-DTW (dctts_mcd_dtw): back-pointers (sum nx_b ny_b bytes), per-pair lengths and offsets (4B int64), the cepstra
    // of pairs too long for shared memory, and rows 1 .. n_mels - 1 of the DCT-II matrix (uploaded at the first call)
    struct { DevBuf bp, meta, cep, dct; } mcd;
    DevBuf join_meta;             // dctts_join_rows: each piece's text and pause (2P ints), then each text's first piece (K + 1)
    DevBuf lbuf;                  // (B, N) ids staging for the host entry point
    DevBuf zbuf;                  // (B, 4T, F) staging for the host entry point
    DevBuf plane[4];              // tensor-core path activations: {hi,lo} x ping-pong, rows x 1032 fp16
    DevBuf in_inv;                // (B) inverse per-utterance scales of a network input's planes (launch_f32_to_planes_scaled)
    DevBuf attpl[6];              // wgmma attention operands: Q, K planes and transposed V planes ({hi,lo} each)
    DevBuf arpl[10];              // AR decode planes: R (B,T,2d) and four AudioDec outputs (B,T,d), {hi,lo} each

    // training step (Text2Mel, reference train.py mode "train"): see the "training" section below
    struct TrainLayer {
        // rows / L / L_in are this step's extents (train_set_shape); pre / out point at capacity-sized slices
        LayerDev* l = nullptr; int li = 0; long long rows = 0; int L = 0, L_in = 0, ld_out = 0; const float* in = nullptr; int ld_in = 0;
        float* pre = nullptr; float* out = nullptr; int extra_shift = 0; bool need_dgrad = true;
        float *dW = nullptr, *dbias = nullptr, *dg1 = nullptr, *db1 = nullptr, *dg2 = nullptr, *db2 = nullptr;
        GemmTcSlots tc_slots;      // abs-max slots of this block's input and weights, set by the forward GEMM of the current step
    };
    struct TrainTensor { float* p; float* g; float* m; float* v; long long n; int layout, d0, d1, d2, ld; };
    struct {
        bool ready = false; int B = 0, num = 1, T_in = 0; float rate = 0.f;   // T_in: capacity in mel frames given at init (num = 1: hp.max_T)
        int N_cap = 0, T_cap = 0;                               // the workspace's capacity: init's (max_N, T_in), grown by dctts_train_reserve
        std::vector<TrainLayer> layers;
        std::map<std::string, TrainTensor> tensors;            // by TF variable name
        DevBuf pre, out, emb, R, align, dS, gbuf[4], dy, wT, zeros, gts, sums, ids, grads, mom, vel, entries;
        long long n_grad = 0; int n_entries = 0; float* d_table = nullptr;
        DevBuf tc_a_hi, tc_a_lo, tc_b_hi, tc_b_lo, tc_slots;    // operand planes of the wgmma training GEMMs (kernels_gemm_tc.cu)
        GemmTcWs tc;
        // ordered sums (option train_deterministic): partials of the largest launch at the capacity, allocated while the option is on
        DevBuf ord_part, ord_dpart; size_t ord_floats = 0; OrderedWs ord;
        int first[3] = {0, 0, 0}, last[3] = {0, 0, 0};         // layer index ranges: TextEnc, AudioEnc, AudioDec
    } tr;

    // vocoder (Griffin-Lim) state
    struct { int hop = 275, win = 1102, n_iter = 50; float power = 1.5f, max_db = 100.f, ref_db = 20.f; double preemph = 0.97; } voc;
    DevBuf feat_melw, feat_range, feat_tw, feat_window, feat_wss;   // feature extraction tables (dctts_get_spectrograms)
    DevBuf feat_seg;                                                // per-utterance segment tables of a feature batch
    DevBuf rs_win, rs_tab;                                          // resampling: kaiser_best filter, per-call tables
    int feat_sr = 0, feat_win = 0;
    DevBuf voc_S, voc_X, voc_frames, voc_mse, voc_tw, voc_window, voc_wss, voc_deemph;
    DevBuf voc_wsq, voc_len;                      // squared window row (n_fft), per-utterance frame counts (ragged call)
    DevBuf voc_E, voc_part;                       // fast Griffin-Lim: previous raw estimate (B, T, F), convergence partials
    int voc_tables_T = 0, voc_tables_win = 0, voc_tables_hop = 0;
    // co-resident 16-CTA clusters of the 144-column block kernel (the F = 2049 conv1d blocks), -1 until first needed;
    // when none fits, why those blocks run on the fp32 kernels
    int tc16_clusters = -1;
    std::string tc16_why;

    // AR decode graph
    cudaGraphExec_t ar_exec = nullptr;
    int ar_B = 0;
    bool ar_path = false;         // the captured step advances along pathbuf instead of to its own argmax
    int64_t ar_nodes = 0;

    int tensor_path = 1;          // wgmma blocks wherever they apply; 0 forces the fp32 CUDA-core kernels
    int64_t launches = 0;

    // kernel-variant switches (dctts_set_option); the defaults are the measured-best configuration
    struct Options {
        int tc_occ2 = 0;          // 1: two-stage ring on launches wider than the device
        int tc_mcast = 1;         // TMA multicast of the activation tile across the cluster
        int tc_resid_tma = 1;     // hc: residual in / planes out through TMA
        int tc_debug = 0;         // progress markers + in-kernel cycle stamps (synchronising)
        int fused_ln = 0;         // graph decode: split-K GEMM and LN epilogue in one launch
        int decode_prof = 0;      // persistent decode: record SM-clock lap timers of cluster 0 / rank 0 (dctts_decode_profile)
        int decode_force_prepass = 0;   // persistent decode, measurement / test only: every utterance recomputes its receptive field at every frame j >= 1
        int decode_mode = 1;      // 1 = persistent cluster kernel (kernels_decode.cu), 0 = one CUDA graph per frame (round-1 path)
        int train_probe = 0;      // measurement only (tools/bench_train.py --probe): the training GEMMs fetch their operands but issue no MMA
        int train_tc = 7;         // training GEMMs on wgmma, bit mask: 1 forward conv, 2 data gradient, 4 weight gradient; 0 = fp32 CUDA-core kernels
        int train_deterministic = 0;   // 1: the training step's sums in a fixed order (kernels_ordered.cu): a seeded run repeats bit for bit
        int chain_history = 0;    // test aid: the full-sequence chains copy every block's rows for dctts_chain_history
        int decode_group = 0;     // measurement: utterances per persistent-decode cluster (1..5); 0 = decode_group's rule
        int decode_timing = 0;    // measurement: CUDA events around every persistent-decode launch (dctts_get_option "decode_last_us")
    } opt;

    // the open synthesis stream (dctts_synth_stream_open), or null: it owns the decode workspace until it is closed
    dctts_synth_stream_s* synth = nullptr;

    // persistent decode (kernels_decode.cu)
    struct {
        bool ok = false;          // stream packed, geometry supported, 16-CTA clusters schedulable
        bool tables_ok = false;   // geometry supported: the tables are built and the stream allocated
        bool commit_ok = false;   // ok / why as commit left them: what a refresh restores
        std::string commit_why;
        DecParams tab{};          // layer / chunk tables (+ parameter pointers); per-call fields filled by text2mel_generate
        DevBuf wstream, lnp, scr, stats, pfinal, prof, pl, frames;
        int max_clusters = 0;
        std::string why;          // why not ok
        int last_moved_frames = -1, last_moved_utt = -1, last_clusters = 0;
        int last_frames = -1;     // frames the last generation executed, summed over clusters (-1: none yet)
        bool frames_pending = false;   // last_frames is still in `frames` (per cluster) on the device
        cudaEvent_t ev[2] = {nullptr, nullptr};   // option decode_timing: around the last persistent-decode launch
        bool timed = false;

    } dec;

    // What dctts_decode_history may read: set by a generation without the final attention pass, cleared by every other
    // writer of kv, rbuf, ae_out, ad_out, ybuf or the AR planes (and by a workspace growth, which reallocates them)
    struct {
        bool ok = false;
        int B = 0;                // utterances of that generation
        unsigned planes_only = 0; // bit i: AudioDec block i wrote only its split planes (arpl[i + 1]), not ad_out[i]
    } hist;

    // What dctts_chain_history may read (option chain_history): copies of the rows the last full-sequence chains left,
    // made device to device as they ran.  Per network (CH_TEXTENC .. CH_ATTENTION): rec[0] the first block's input as the
    // kernel read it, rec[1 + i] block i's output; the attention's rec[1] is R.  A record holds fp32 rows or a plane pair.
    struct ChainRec { DevBuf a, b; int B = 0, L = 0, C = 0, ld = 0; bool planes = false, scaled = false; DevBuf inv; };
    struct {
        std::vector<ChainRec> rec[5];
        unsigned nets = 0;        // bit n: network n's records belong to the last writer
        std::string why = "no full-sequence chain has run since the handle was created";   // why a network is not readable
    } chist;

    // the device buffers free themselves after this body: the graph that points into them goes first
    ~dctts_handle_s() {
        if (ar_exec) cudaGraphExecDestroy(ar_exec);
        if (copy_stream) { cudaStreamDestroy(copy_stream); for (auto e : chunk_done) if (e) cudaEventDestroy(e); }
        if (path_uploaded) { cudaEventSynchronize(path_uploaded); cudaEventDestroy(path_uploaded); }
        for (auto e : dec.ev) if (e) cudaEventDestroy(e);
        if (path_pinned) cudaFreeHost(path_pinned);
        if (stream) cudaStreamDestroy(stream);
    }
};

namespace dctts::api {

using H = dctts_handle_s;

struct Launch {
    H* h; cudaStream_t s;
    std::vector<cudaEvent_t>* evs = nullptr;     // profile mode: one event after every kernel
    void count(int n = 1) {
        h->launches += n;
        if (evs) {
            cudaEvent_t e;
            CUDA_CHECK(cudaEventCreate(&e));
            CUDA_CHECK(cudaEventRecord(e, s));
            evs->push_back(e);
        }
    }
};

template <class Fn>
int guarded(dctts_handle h, Fn&& fn) {
    if (!h) { g_create_error = "null handle"; return 1; }
    try {
        CUDA_CHECK(cudaSetDevice(h->device));
        fn();
        CUDA_CHECK(cudaGetLastError());
        return 0;
    } catch (const std::exception& e) {
        h->err = e.what();
        cudaGetLastError();
        return 2;
    } catch (...) {
        h->err = "unknown failure";
        return 3;
    }
}

// Per-utterance integers from the caller's host memory, checked before anything is launched: values[b] in [lo, hi] for
// b < B or, with `counts`, the first counts[b] values of row b of the (B, ld) array `values`, one per frame.  The first
// value outside fails the call, naming its utterance (and frame): "<fn>: utterance <b> has <what> <v> outside [lo, hi]".
inline void require_each(const std::string& fn, const char* what, const int* values, int B, long long lo, long long hi,
                         const int* counts = nullptr, size_t ld = 0) {
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < (counts ? counts[b] : 1); ++j) {
            const int v = counts ? values[(size_t)b * ld + j] : values[b];
            if (v < lo || v > hi)
                throw std::runtime_error(fn + ": utterance " + std::to_string(b) + " has " + what + " " + std::to_string(v) +
                                         (counts ? " at frame " + std::to_string(j) : std::string()) + " outside [" +
                                         std::to_string(lo) + ", " + std::to_string(hi) + "]");
        }
}

// Entry points that write the decode workspace, the weights or grow buffers are refused while a synthesis stream is open:
// its decode and SSRN windows are still reading them.
inline void require_no_synth_stream(const H* h, const std::string& what) {
    if (h->synth)
        throw std::runtime_error(what + ": a synthesis stream is open on this handle (dctts_synth_stream_open); close it first");
}

// NULL means the legacy default stream (what torch's default stream is), so calls made from a
// torch program are ordered with the surrounding torch work without extra synchronisation.
inline cudaStream_t S(dctts_handle, void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ---------------------------------------------------------------------------- called across stages
void build_tables(H* h);                                                          // api_params.cu
void pack_weights(H* h, cudaStream_t s);
void mark_synthesis_stale(H* h);
std::vector<int> audiodec_rows(const std::vector<LayerDev>& net, int T);          // api_synth.cu
void settle_decode_counts(H* h);
void chist_clear(H* h, const std::string& why);                                  // the chain history is stale
void drop_ar_graph(H* h);
void synth_stream_free(dctts_synth_stream_s* ss);                                 // close without outputs (dctts_destroy)
void run_attention(Launch& lc, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                   RowWin win, int N, const int* pma, float* R, float* align, long long* maxatt,
                   int* p_next, int* p_hist, Planes Rpl = Planes{});
void run_attention_tc(Launch& lc, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, int B, int T,
                      int N, const int* pma, float* R, float* align, long long* maxatt, Planes Rpl);

}  // namespace dctts::api
