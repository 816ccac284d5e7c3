// dctts_api.cu -- the handle's life cycle, its options and the pass-throughs of the C-ABI (include/dctts.h).
#include "api_internal.cuh"

std::string dctts::api::g_create_error;

namespace {

// Kernel-variant switches: every value selects a parity-tested code path (tests/test_gpu_variants.py); the defaults are the
// measured-best configuration.  Replaces the environment variables of round 1, which froze at first use.
using OptionSlot = int H::Options::*;
struct Option { const char* name; OptionSlot slot; int max; };
const Option kOptions[] = {
    {"tc_occ2", &H::Options::tc_occ2, 2},         {"tc_mcast", &H::Options::tc_mcast, 2},
    {"tc_resid_tma", &H::Options::tc_resid_tma, 2}, {"tc_debug", &H::Options::tc_debug, 2},
    {"fused_ln", &H::Options::fused_ln, 2},       {"decode_mode", &H::Options::decode_mode, 2},
    {"decode_prof", &H::Options::decode_prof, 2}, {"decode_force_prepass", &H::Options::decode_force_prepass, 2},
    {"train_tc", &H::Options::train_tc, 7},       {"train_probe", &H::Options::train_probe, 2},
    {"train_deterministic", &H::Options::train_deterministic, 1},
    {"chain_history", &H::Options::chain_history, 1},
    {"decode_group", &H::Options::decode_group, 5},  {"decode_timing", &H::Options::decode_timing, 1},
};

const Option* find_option(const char* name) {
    for (const Option& o : kOptions)
        if (name && std::strcmp(name, o.name) == 0) return &o;
    return nullptr;
}

}  // namespace

extern "C" {

const char* dctts_version(void) { return "dc_tts_b200 0.1.0 (sm_90a)"; }

const char* dctts_last_error(dctts_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int dctts_create(const dctts_hparams* hp, int device, dctts_handle* out) {
    if (!hp || !out) { g_create_error = "dctts_create: null argument"; return 1; }
    try {
        int ndev = 0;
        CUDA_CHECK(cudaGetDeviceCount(&ndev));
        if (device < 0 || device >= ndev) throw std::runtime_error("dctts_create: no such CUDA device (no CPU fallback exists)");
        cudaDeviceProp prop;
        CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0) throw std::runtime_error("dctts_create: this library is built for sm_90a (H100) only");
        if (hp->d > 256 || hp->d % 8 || hp->e % 4 || hp->max_N < 1 || hp->r != 4)
            throw std::runtime_error("dctts_create: unsupported hyper-parameters");
        std::unique_ptr<dctts_handle_s> h(new dctts_handle_s());
        h->hp = *hp; h->device = device; h->F = 1 + hp->n_fft / 2; h->num_sms = prop.multiProcessorCount;
        CUDA_CHECK(cudaSetDevice(device));
        CUDA_CHECK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        build_tables(h.get());
        h->tickets.ensure(64 * sizeof(int));
        CUDA_CHECK(cudaMemset(h->tickets.p, 0, 64 * sizeof(int)));
        h->pack_max.ensure(PACK_MAXL * sizeof(unsigned));
        *out = h.release();
        return 0;
    } catch (const std::exception& e) {
        g_create_error = e.what();
        cudaGetLastError();
        return 2;
    }
}

int dctts_destroy(dctts_handle h) {
    if (!h) return 1;
    cudaSetDevice(h->device);
    if (h->synth) synth_stream_free(h->synth);      // waits for its decode
    cudaDeviceSynchronize();
    delete h;
    return 0;
}

int64_t dctts_launch_count(dctts_handle h) { return h ? h->launches : -1; }

// CRC-32C (polynomial 0x1EDC6F41, reflected 0x82F63B78), slicing-by-8 on the host.
uint32_t dctts_crc32c(uint32_t crc, const void* data, int64_t n) {
    struct Table {
        uint32_t T[8][256];
        Table() {
            for (uint32_t i = 0; i < 256; ++i) {
                uint32_t c = i;
                for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0x82F63B78u : (c >> 1);
                T[0][i] = c;
            }
            for (uint32_t i = 0; i < 256; ++i)
                for (int t = 1; t < 8; ++t) T[t][i] = (T[t - 1][i] >> 8) ^ T[0][T[t - 1][i] & 0xffu];
        }
    };
    static const Table tab;                 // C++11: initialised once, thread-safe
    const auto& T = tab.T;
    const uint8_t* p = static_cast<const uint8_t*>(data);
    uint32_t c = ~crc;
    while (n > 0 && (reinterpret_cast<uintptr_t>(p) & 7u)) { c = (c >> 8) ^ T[0][(c ^ *p++) & 0xffu]; --n; }
    while (n >= 8) {
        uint64_t v;
        memcpy(&v, p, 8);
        const uint32_t lo = (uint32_t)v ^ c, hi = (uint32_t)(v >> 32);
        c = T[7][lo & 0xffu] ^ T[6][(lo >> 8) & 0xffu] ^ T[5][(lo >> 16) & 0xffu] ^ T[4][lo >> 24] ^
            T[3][hi & 0xffu] ^ T[2][(hi >> 8) & 0xffu] ^ T[1][(hi >> 16) & 0xffu] ^ T[0][hi >> 24];
        p += 8; n -= 8;
    }
    while (n-- > 0) c = (c >> 8) ^ T[0][(c ^ *p++) & 0xffu];
    return ~c;
}

int dctts_set_option(dctts_handle h, const char* name, int32_t value) {
    return guarded(h, [&] {
        if (name && std::string(name) == "pdl") { pdl_enabled() = value != 0; return; }     // process-wide launch attribute
        const Option* o = find_option(name);
        REQUIRE(o, "dctts_set_option: unknown option");
        REQUIRE(value >= 0 && value <= o->max, "dctts_set_option: value out of range");
        if (o->slot == &H::Options::decode_mode && value == 1 && !h->dec.ok && h->committed)
            throw std::runtime_error("dctts_set_option: persistent decode unavailable: " + h->dec.why);
        int& slot = h->opt.*o->slot;
        if (slot != value && h->ar_exec) {                   // the captured AR step bakes the variant in
            CUDA_CHECK(cudaDeviceSynchronize());
            drop_ar_graph(h);
        }
        slot = value;
    });
}

int dctts_get_option(dctts_handle h, const char* name, int32_t* value) {
    return guarded(h, [&] {
        REQUIRE(value, "dctts_get_option: null output");
        if (name && std::string(name) == "pdl") { *value = pdl_enabled() ? 1 : 0; return; }
        if (name && std::string(name) == "decode_available") { *value = h->dec.ok ? 1 : 0; return; }
        if (name && std::string(name) == "decode_max_clusters") { *value = h->dec.max_clusters; return; }   // co-resident 16-CTA clusters
        if (name && std::string(name) == "decode_last_frames") {     // frames the last generation executed, summed over clusters
            REQUIRE(h->dec.last_frames >= 0 || h->dec.frames_pending, "dctts_get_option(decode_last_frames): no generation has run");
            settle_decode_counts(h);
            *value = h->dec.last_frames;
            return;
        }
        if (name && std::string(name) == "decode_last_us") {        // option decode_timing: the last persistent decode's GPU time
            REQUIRE(h->dec.timed, "dctts_get_option(decode_last_us): no persistent decode has run with option decode_timing");
            CUDA_CHECK(cudaEventSynchronize(h->dec.ev[1]));
            float ms = 0.f;
            CUDA_CHECK(cudaEventElapsedTime(&ms, h->dec.ev[0], h->dec.ev[1]));
            *value = (int32_t)std::lround(1e3 * ms);
            return;
        }
        if (name && std::string(name) == "ssrn_tc_available") {     // every SSRN block has a wgmma kernel (needs committed parameters)
            REQUIRE(h->committed, "dctts_get_option(ssrn_tc_available): parameters not committed");
            REQUIRE(h->tc16_why.empty(), "dctts_get_option(ssrn_tc_available): " + h->tc16_why);
            bool ok = !h->ssrn.empty();
            for (const auto& l : h->ssrn) ok = ok && l.tc.ok;
            *value = ok ? 1 : 0;
            return;
        }
        const Option* o = find_option(name);
        REQUIRE(o, "dctts_get_option: unknown option");
        *value = h->opt.*o->slot;
    });
}

int dctts_malloc(dctts_handle h, void** ptr, int64_t bytes) {
    return guarded(h, [&] { REQUIRE(ptr && bytes > 0, "dctts_malloc: bad arguments"); CUDA_CHECK(cudaMalloc(ptr, (size_t)bytes)); });
}
int dctts_free(dctts_handle h, void* ptr) { return guarded(h, [&] { CUDA_CHECK(cudaFree(ptr)); }); }
int dctts_memcpy_h2d(dctts_handle h, void* dst, const void* src, int64_t bytes, void* stream) {
    return guarded(h, [&] { CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyHostToDevice, S(h, stream))); });
}
int dctts_memcpy_d2h(dctts_handle h, void* dst, const void* src, int64_t bytes, void* stream) {
    return guarded(h, [&] { CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToHost, S(h, stream))); });
}
int dctts_malloc_host(dctts_handle h, void** ptr, int64_t bytes) {
    return guarded(h, [&] { REQUIRE(ptr && bytes > 0, "dctts_malloc_host: bad arguments"); CUDA_CHECK(cudaMallocHost(ptr, (size_t)bytes)); });
}
int dctts_free_host(dctts_handle h, void* ptr) { return guarded(h, [&] { CUDA_CHECK(cudaFreeHost(ptr)); }); }
int dctts_stream_sync(dctts_handle h, void* stream) { return guarded(h, [&] { CUDA_CHECK(cudaStreamSynchronize(S(h, stream))); }); }

}  // extern "C"
