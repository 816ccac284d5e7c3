// api_audio.cu -- the Griffin-Lim vocoder, on-device feature extraction (load_spectrograms) and resampling.
#include "api_internal.cuh"

namespace {

// The STFT kernels exist for n_fft 1024, 2048 and 4096 (F = 513, 1025, 2049)
void require_fft_size(const H* h, const std::string& fn) {
    const int n_fft = 2 * (h->F - 1);
    REQUIRE(voc_fft_size_ok(n_fft), fn + ": n_fft = " + std::to_string(n_fft) + " has no STFT kernel (supported: 1024, 2048, 4096)");
    REQUIRE(h->voc.win <= n_fft, fn + ": win_length " + std::to_string(h->voc.win) + " exceeds n_fft = " + std::to_string(n_fft) +
                                 " (dctts_set_vocoder_params)");
}

// librosa.effects.trim(y)[1] from the per-frame mean squares: frames within 60 dB of the loudest one
void trim_from_mse(const float* m, int nfr, int Ly, int32_t* out) {
    float mx = 0.f;
    for (int f = 0; f < nfr; ++f) mx = std::max(mx, m[f]);
    const double ref = 10.0 * std::log10(std::max(1e-10, (double)mx));
    int first = -1, last = -1;
    for (int f = 0; f < nfr; ++f) {
        const double db = 10.0 * std::log10(std::max(1e-10, (double)m[f])) - ref;
        if (db > -60.0) { if (first < 0) first = f; last = f; }
    }
    out[0] = first < 0 ? 0 : first * 512;
    out[1] = first < 0 ? 0 : std::min(Ly, (last + 1) * 512);
}

// The mel basis, FFT twiddles and Hann window of the feature kernels, rebuilt when the sample rate or window changes.
void feat_tables(H* h, int sample_rate, cudaStream_t s) {
    const int win = h->voc.win, hop = h->voc.hop;
    if (h->feat_sr == sample_rate && h->feat_win == win) return;
    std::vector<float> w; std::vector<int> range;
    feat_make_mel_basis(sample_rate, h->hp.n_fft, h->hp.n_mels, w, range);
    h->feat_melw.ensure(w.size() * sizeof(float)); h->feat_range.ensure(range.size() * sizeof(int));
    const int n_fft = 2 * (h->F - 1);
    h->feat_tw.ensure(n_fft * sizeof(float2)); h->feat_window.ensure(win * sizeof(float)); h->feat_wss.ensure(n_fft * sizeof(float));
    CUDA_CHECK(cudaMemcpyAsync(h->feat_melw.p, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_CHECK(cudaMemcpyAsync(h->feat_range.p, range.data(), range.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    voc_make_tables(n_fft, h->feat_tw.as<float2>(), h->feat_window.as<float>(), h->feat_wss.as<float>(), 1, win, hop, s);   // synchronises
    h->feat_sr = sample_rate; h->feat_win = win;
}

// The arguments of feat_run for `frames` STFT frames of B trimmed utterances (seg_dev: B + 1 device entries), with the
// handle's tables and vocoder parameters: mag (B, r T_b, F), mel (B, T_b, n_mels)
FeatArgs feat_args(const H* h, const void* wav, int dtype, const FeatSeg* seg_dev, int B, long long frames, float* mel, float* mag,
                   int T_b, int r) {
    FeatArgs a{};
    a.wav = wav; a.dtype = dtype; a.seg = seg_dev; a.B = B; a.frames = (int)frames;
    a.mag = mag; a.mel = mel; a.mag_rows = r * T_b; a.mel_rows = T_b; a.r = r;
    a.melw = h->feat_melw.as<float>(); a.melrange = h->feat_range.as<int>(); a.tw = h->feat_tw.as<float2>();
    a.window = h->feat_window.as<float>(); a.F = h->F; a.n_mels = h->hp.n_mels; a.win = h->voc.win; a.hop = h->voc.hop;
    a.preemph = (float)h->voc.preemph; a.ref_db = h->voc.ref_db; a.max_db = h->voc.max_db;
    return a;
}

// load_spectrograms (utils.py:147-162) for B utterances packed back to back in `wav` (offsets: B + 1 host sample
// offsets), reduced by r and padded with zeros to the batch's longest member: mel (B, T_b, n_mels), mag (B, r T_b, F).
// r = 1 is get_spectrograms (utils.py:20-65): every frame, T_b = T for one utterance.  Two kernels whatever B is:
// the trim energies of every utterance (one copy back, thresholded on the host: the call's one synchronisation), then
// the features, one CTA per STFT frame of the flattened batch.  Nothing is written to mel or mag unless every
// utterance survives trimming and T_b <= t_capacity.
void feat_batch(H* h, const char* who, const void* wav, int dtype, const int64_t* offsets, int B, int sample_rate, float* mel,
                float* mag, int t_capacity, int r, int32_t* t_host, int32_t* trim_host, int32_t* T_b_out, cudaStream_t s) {
    const std::string fn(who);
    REQUIRE(wav && offsets && mel && mag && B >= 1 && (dtype == 0 || dtype == 1) && sample_rate > 0 && t_capacity >= 1 && r >= 1,
            fn + ": bad arguments");
    require_fft_size(h, fn);
    std::vector<FeatSeg> seg(2 * (size_t)(B + 1));
    FeatSeg* mseg = seg.data();                     // whole utterances, frames of the trim energies
    FeatSeg* fseg = seg.data() + B + 1;             // trimmed utterances, STFT frames
    long long nfr_total = 0;
    for (int b = 0; b < B; ++b) {
        const long long n = offsets[b + 1] - offsets[b];
        REQUIRE(offsets[b] >= 0 && n >= 2 && n < (1ll << 30),
                fn + ": utterance " + std::to_string(b) + " has " + std::to_string(n) + " samples (need 2 to 2^30)");
        mseg[b] = FeatSeg{offsets[b], (int)n, (int)nfr_total};
        nfr_total += 1 + n / 512;
    }
    REQUIRE(nfr_total < (1ll << 31), fn + ": batch too long");
    mseg[B] = FeatSeg{0, 0, (int)nfr_total};
    feat_tables(h, sample_rate, s);
    const int F = h->F, hop = h->voc.hop, n_mels = h->hp.n_mels;
    h->feat_seg.ensure(seg.size() * sizeof(FeatSeg));
    FeatSeg* seg_dev = h->feat_seg.as<FeatSeg>();
    h->voc_mse.ensure((size_t)nfr_total * sizeof(float));
    // librosa.effects.trim (utils.py:36): frame energies on the device, threshold on the host
    CUDA_CHECK(cudaMemcpyAsync(seg_dev, mseg, (B + 1) * sizeof(FeatSeg), cudaMemcpyHostToDevice, s));
    feat_frame_mse(wav, dtype, seg_dev, B, (int)nfr_total, h->voc_mse.as<float>(), s);
    h->launches += 1;
    CUDA_CHECK(cudaGetLastError());
    std::vector<float> mse((size_t)nfr_total);
    CUDA_CHECK(cudaMemcpyAsync(mse.data(), h->voc_mse.p, mse.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    long long frames = 0;
    int T_b = 0, longest = 0;
    bool padded = false;
    std::vector<int> T(B);
    for (int b = 0; b < B; ++b) {
        int se[2];
        trim_from_mse(mse.data() + mseg[b].f0, 1 + mseg[b].len / 512, mseg[b].len, se);
        if (trim_host) { trim_host[2 * b] = se[0]; trim_host[2 * b + 1] = se[1]; }
        const int len = se[1] - se[0];
        REQUIRE(len >= 2, fn + ": utterance " + std::to_string(b) + " has nothing left after trimming (silent input)");
        T[b] = 1 + len / hop;
        const int t = (T[b] + r - 1) / r;           // reduced rows after padding T to a multiple of r
        if (t_host) t_host[b] = t;
        if (t > T_b) { T_b = t; longest = b; }
        fseg[b] = FeatSeg{mseg[b].src + se[0], len, (int)frames};
        frames += T[b];
    }
    for (int b = 0; b < B; ++b) padded = padded || T[b] != r * T_b;
    fseg[B] = FeatSeg{0, 0, (int)frames};
    if (T_b_out) *T_b_out = T_b;
    REQUIRE(T_b <= t_capacity, fn + ": output buffers too small: utterance " + std::to_string(longest) + " needs " +
                               std::to_string(T_b) + " rows, t_capacity is " + std::to_string(t_capacity));
    REQUIRE(frames < (1ll << 31), fn + ": batch too long");
    CUDA_CHECK(cudaMemcpyAsync(seg_dev + B + 1, fseg, (B + 1) * sizeof(FeatSeg), cudaMemcpyHostToDevice, s));
    if (padded) {                                   // bucket padding (data_load.py:128, dynamic_pad) and utils.py:154-158
        CUDA_CHECK(cudaMemsetAsync(mel, 0, (size_t)B * T_b * n_mels * sizeof(float), s));
        CUDA_CHECK(cudaMemsetAsync(mag, 0, (size_t)B * r * T_b * F * sizeof(float), s));
    }
    feat_run(feat_args(h, wav, dtype, seg_dev + B + 1, B, frames, mel, mag, T_b, r), s);
    h->launches += 1;
    CUDA_CHECK(cudaGetLastError());
}

// The handle's vocoder buffers and tables sized for (B, T) and its parameters; the caller sets mag, wav and n_iter.
VocoderArgs voc_args(H* h, const char* fn, int B, int T, cudaStream_t s) {
    REQUIRE(B >= 1 && T >= 2, std::string(fn) + ": need B >= 1 and T >= 2 frames, got B = " + std::to_string(B) + ", T = " +
                              std::to_string(T));
    require_fft_size(h, fn);
    const int F = h->F, n_fft = 2 * (F - 1), win = h->voc.win, hop = h->voc.hop, Ly = hop * (T - 1), nfr = 1 + Ly / 512;
    const size_t n = (size_t)B * T * F;
    h->voc_S.ensure(n * sizeof(float)); h->voc_X.ensure(n * sizeof(float2));
    h->voc_frames.ensure((size_t)B * T * win * sizeof(float)); h->voc_mse.ensure((size_t)B * nfr * sizeof(float));
    h->voc_deemph.ensure(voc_deemph_scratch_bytes(B, T, hop));
    if (h->voc_tables_T != T || h->voc_tables_win != win || h->voc_tables_hop != hop) {
        h->voc_tw.ensure(n_fft * sizeof(float2)); h->voc_window.ensure(win * sizeof(float));
        h->voc_wss.ensure((size_t)(n_fft + hop * (T - 1)) * sizeof(float)); h->voc_wsq.ensure(n_fft * sizeof(float));
        voc_make_tables(n_fft, h->voc_tw.as<float2>(), h->voc_window.as<float>(), h->voc_wss.as<float>(), T, win, hop, s,
                        h->voc_wsq.as<float>());
        CUDA_CHECK(cudaGetLastError());
        h->voc_tables_T = T; h->voc_tables_win = win; h->voc_tables_hop = hop;
    }
    VocoderArgs a{};
    a.S = h->voc_S.as<float>(); a.X = h->voc_X.as<float2>(); a.frames = h->voc_frames.as<float>();
    a.mse = h->voc_mse.as<float>(); a.tw = h->voc_tw.as<float2>(); a.window = h->voc_window.as<float>();
    a.wss = h->voc_wss.as<float>(); a.wsq = h->voc_wsq.as<float>(); a.deemph = h->voc_deemph.as<double>(); a.B = B; a.T = T; a.F = F; a.win = win; a.hop = hop;
    a.n_iter = h->voc.n_iter;
    a.max_db = h->voc.max_db; a.ref_db = h->voc.ref_db; a.power = h->voc.power; a.preemphasis = h->voc.preemph;
    return a;
}

// librosa.effects.trim from the device frame energies a.mse (B, 1 + Ly / 512): frames within 60 dB of the loudest.
// T_host (optional): the frame count of each utterance of a ragged call, whose energies cover its own 1 + Ly_b / 512
// frames.  Synchronises s.
void voc_trims(const VocoderArgs& a, int32_t* trim_host, cudaStream_t s, const int32_t* T_host = nullptr) {
    const int Ly = a.hop * (a.T - 1), nfr = 1 + Ly / 512;
    std::vector<float> mse((size_t)a.B * nfr);
    CUDA_CHECK(cudaMemcpyAsync(mse.data(), a.mse, mse.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    if (trim_host)
        for (int b = 0; b < a.B; ++b) {
            const int Lyb = T_host ? a.hop * (T_host[b] - 1) : Ly;
            trim_from_mse(mse.data() + (size_t)b * nfr, 1 + Lyb / 512, Lyb, trim_host + 2 * b);
        }
}

// The fast Griffin-Lim weight alpha = momentum / (1 + momentum), formed in float64 and rounded to float32 as numpy does
// when it multiplies a complex64 array by a Python float
float momentum_alpha(const std::string& fn, double momentum) {
    REQUIRE(std::isfinite(momentum) && momentum >= 0.0,
            fn + ": momentum must be finite and >= 0, got " + std::to_string(momentum));
    return (float)(momentum / (1.0 + momentum));
}

// The three spectrogram2wav entry points: Griffin-Lim on mag (B, T, F) into wav, with the fast Griffin-Lim update when
// momentum rounds to a non-zero alpha, per-utterance frame counts when lengths_host is given and the spectral
// convergence of every iteration when convergence is given.  fn names the entry point in every error message.
void griffin_lim(H* h, const char* fn, const float* mag, int B, int T, const int32_t* lengths_host, int n_iter,
                 double momentum, float* wav, int32_t* trim_host, double* convergence, cudaStream_t s) {
    const float alpha = momentum_alpha(fn, momentum);
    if (lengths_host) require_each(fn, "frame count", lengths_host, B, 2, T);
    VocoderArgs a = voc_args(h, fn, B, T, s);
    a.mag = mag; a.wav = wav;
    if (n_iter >= 0) a.n_iter = n_iter;
    if (lengths_host) {
        h->voc_len.ensure((size_t)B * sizeof(int));
        CUDA_CHECK(cudaMemcpyAsync(h->voc_len.p, lengths_host, (size_t)B * sizeof(int), cudaMemcpyHostToDevice, s));
        a.lengths = h->voc_len.as<int>();
    }
    if (alpha != 0.f) {                 // est_{-1} = 0; a momentum that rounds to alpha = 0 is the plain update
        const size_t n = (size_t)B * T * a.F * sizeof(float2);
        h->voc_E.ensure(n);
        CUDA_CHECK(cudaMemsetAsync(h->voc_E.p, 0, n, s));
        a.E = h->voc_E.as<float2>(); a.alpha = alpha;
    }
    if (convergence) {
        h->voc_part.ensure((size_t)(a.n_iter + 1) * B * T * sizeof(float));
        a.part = h->voc_part.as<float>(); a.conv = convergence;
    }
    voc_run(a, s);
    h->launches += voc_launches_per_call(a.n_iter, convergence != nullptr);
    CUDA_CHECK(cudaGetLastError());
    voc_trims(a, trim_host, s, lengths_host);
}

}  // namespace

// Look-ahead margin of the streaming vocoder, in frames: a push commits up to the support start of frame t_r - M, t_r the
// first frame whose window reaches the prefix's reflected tail.  The smallest of {0, 2, 4, 8} whose streamed spectral
// convergence stays within 1.5x of whole-signal Griffin-Lim (DESIGN.md section 8i)
constexpr int VOC_STREAM_MARGIN = 0;

// One vocoder stream: the Griffin-Lim state of B utterances of up to T frames, the de-emphasised waveform they committed,
// and the host's account of each utterance (frames received, samples committed, final).
struct dctts_vocoder_stream_s {
    H* h = nullptr;
    cudaStream_t s = nullptr;
    int B = 0, T = 0, F = 0, n_iter = 0;
    float alpha = 0.f;
    DevBuf S, X, E, frames, y, wav, mse, tw, window, wss, wsq, deemph, state, meta;
    std::vector<int> A, c, ended;
    VocoderArgs args;          // the buffers and tables; each push fills the per-step bounds
};

namespace {

// Window support of frame t in the centre-trimmed signal: [hop t + a0, hop t + a1)
struct VocSupport { int a0, a1; };
VocSupport voc_support(int n_fft, int win) {
    const int lpad = (n_fft - win) / 2;
    return {lpad - n_fft / 2, lpad + win - n_fft / 2};
}

// The first frame whose window reaches a sample >= c: the frames below touch only committed samples
int voc_first_active(int c, int hop, VocSupport w) { return c < w.a1 ? 0 : (c - w.a1) / hop + 1; }

// The committed sample count after a step over A frames from c (tests/ref_stream_vocoder.py: commit_end)
int voc_commit_end(int c, int A, bool final, int hop, VocSupport w) {
    const int Ly = hop * (A - 1);
    if (final) return Ly;
    const int t_r = std::max(0, (Ly - w.a1 + 1 + hop - 1) / hop);     // first frame reading a sample >= Ly (reflected)
    return std::min(Ly, std::max(c, hop * (t_r - VOC_STREAM_MARGIN) + w.a0));
}

void vocoder_stream_open(H* h, int B, int T, int n_iter, double momentum, cudaStream_t s, dctts_vocoder_stream* out) {
    const std::string fn = "dctts_vocoder_stream_open";
    REQUIRE(out, fn + ": out is required");
    REQUIRE(B >= 1 && T >= 2, fn + ": need B >= 1 and T_cap >= 2 frames, got B = " + std::to_string(B) + ", T_cap = " +
                              std::to_string(T));
    require_fft_size(h, fn);
    auto vs = std::make_unique<dctts_vocoder_stream_s>();
    vs->h = h; vs->s = s; vs->B = B; vs->T = T; vs->F = h->F;
    vs->n_iter = n_iter >= 0 ? n_iter : h->voc.n_iter;
    vs->alpha = momentum_alpha(fn, momentum);
    const int F = h->F, n_fft = 2 * (F - 1), win = h->voc.win, hop = h->voc.hop, Ly = hop * (T - 1);
    const size_t n = (size_t)B * T * F;
    vs->S.ensure(n * sizeof(float)); vs->X.ensure(n * sizeof(float2)); vs->E.ensure(n * sizeof(float2));
    vs->frames.ensure((size_t)B * T * win * sizeof(float));
    vs->y.ensure((size_t)B * Ly * sizeof(float)); vs->wav.ensure((size_t)B * Ly * sizeof(float));
    vs->mse.ensure((size_t)B * (1 + Ly / 512) * sizeof(float));
    vs->deemph.ensure(voc_deemph_scratch_bytes(B, T, hop)); vs->state.ensure((size_t)B * sizeof(double));
    vs->meta.ensure((size_t)B * 6 * sizeof(int));
    vs->tw.ensure(n_fft * sizeof(float2)); vs->window.ensure(win * sizeof(float));
    vs->wss.ensure((size_t)(n_fft + Ly) * sizeof(float)); vs->wsq.ensure(n_fft * sizeof(float));
    voc_make_tables(n_fft, vs->tw.as<float2>(), vs->window.as<float>(), vs->wss.as<float>(), T, win, hop, s, vs->wsq.as<float>());
    // est_{-1} = 0 for every frame: a frame's E is written only once it has been active, so this covers every new frame
    CUDA_CHECK(cudaMemsetAsync(vs->E.p, 0, n * sizeof(float2), s));
    CUDA_CHECK(cudaMemsetAsync(vs->y.p, 0, (size_t)B * Ly * sizeof(float), s));
    CUDA_CHECK(cudaMemsetAsync(vs->wav.p, 0, (size_t)B * Ly * sizeof(float), s));
    CUDA_CHECK(cudaMemsetAsync(vs->state.p, 0, (size_t)B * sizeof(double), s));
    VocoderArgs& a = vs->args;
    a = VocoderArgs{};
    a.S = vs->S.as<float>(); a.X = vs->X.as<float2>(); a.frames = vs->frames.as<float>(); a.wav = vs->y.as<float>();
    a.mse = vs->mse.as<float>(); a.tw = vs->tw.as<float2>(); a.window = vs->window.as<float>(); a.wss = vs->wss.as<float>();
    a.wsq = vs->wsq.as<float>(); a.deemph = vs->deemph.as<double>(); a.B = B; a.T = T; a.F = F; a.win = win; a.hop = hop;
    a.n_iter = vs->n_iter; a.max_db = h->voc.max_db; a.ref_db = h->voc.ref_db; a.power = h->voc.power;
    a.preemphasis = h->voc.preemph;
    if (vs->alpha != 0.f) { a.E = vs->E.as<float2>(); a.alpha = vs->alpha; }
    int* m = vs->meta.as<int>();          // lengths, new_lo, frame_lo, sample_lo (B each), span (B int2)
    a.lengths = m; a.new_lo = m + B; a.frame_lo = m + 2 * B; a.sample_lo = m + 3 * B;
    a.span = reinterpret_cast<const int2*>(m + 4 * B); a.state = vs->state.as<double>();
    vs->A.assign(B, 0); vs->c.assign(B, 0); vs->ended.assign(B, 0);
    CUDA_CHECK(cudaGetLastError());
    *out = vs.release();
}

void vocoder_stream_push(dctts_vocoder_stream vs, const float* mag, int R, const int32_t* rows, const int32_t* final_host,
                         float* wav_out, int64_t ld, int32_t* counts) {
    const std::string fn = "dctts_vocoder_stream_push";
    REQUIRE(rows && counts && R >= 0 && (mag || R == 0) && (wav_out || ld == 0) && ld >= 0, fn + ": bad arguments");
    const int B = vs->B, T = vs->T, hop = vs->args.hop, Ly_row = hop * (T - 1);
    const VocSupport w = voc_support(2 * (vs->F - 1), vs->args.win);
    require_each(fn, "row count", rows, B, 0, R);
    // lengths, new_lo, frame_lo, sample_lo, span: utterances without a step get empty ranges
    std::vector<int> m((size_t)B * 6);
    std::vector<int> c_new(vs->c);
    int n_active = 0, n_samples = 0, n_span = 0, stepping = 0;
    for (int b = 0; b < B; ++b) {
        const std::string who = fn + ": utterance " + std::to_string(b);
        const bool fin = final_host && final_host[b];
        REQUIRE(!vs->ended[b] || (rows[b] == 0 && !fin), who + " has had its final push");
        const int A = vs->A[b] + rows[b];
        REQUIRE(A <= T, who + " would have " + std::to_string(A) + " frames, past T_cap = " + std::to_string(T));
        REQUIRE(!fin || A >= 2, who + " ends with " + std::to_string(A) + " frame(s); an utterance needs at least 2");
        m[b] = A; m[B + b] = vs->A[b];
        m[2 * B + b] = T; m[3 * B + b] = Ly_row; m[4 * B + 2 * b] = m[4 * B + 2 * b + 1] = vs->c[b];
        if ((rows[b] > 0 || fin) && A >= 2) {
            const int lo = voc_first_active(vs->c[b], hop, w), Ly = hop * (A - 1);
            c_new[b] = voc_commit_end(vs->c[b], A, fin, hop, w);
            m[2 * B + b] = lo; m[3 * B + b] = vs->c[b]; m[4 * B + 2 * b + 1] = c_new[b];
            n_active = std::max(n_active, A - lo);
            n_samples = std::max(n_samples, Ly - vs->c[b]);
            n_span = std::max(n_span, c_new[b] - vs->c[b]);
            ++stepping;
        }
        REQUIRE(c_new[b] - vs->c[b] <= ld, who + " commits " + std::to_string(c_new[b] - vs->c[b]) + " samples, past ld = " +
                                           std::to_string(ld));
    }
    H* h = vs->h;
    cudaStream_t s = vs->s;
    VocoderArgs a = vs->args;
    a.mag = mag; a.n_new = R; a.n_active = n_active; a.n_samples = n_samples; a.n_span = n_span;
    CUDA_CHECK(cudaMemcpyAsync(vs->meta.p, m.data(), m.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    if (R > 0) { voc_prepare(a, s); h->launches += 1; }
    if (stepping) {
        for (int it = 0; it <= a.n_iter; ++it) {
            voc_istft(a, s);
            if (it < a.n_iter) voc_stft_phase(a, s, it);
        }
        h->launches += 3 * a.n_iter + 2;
    }
    if (n_span > 0) {
        a.deemph_in = vs->y.as<float>(); a.wav = vs->wav.as<float>();
        voc_deemph(a, s);
        h->launches += 3;
    }
    for (int b = 0; b < B; ++b) {
        counts[b] = c_new[b] - vs->c[b];
        if (counts[b] > 0)
            CUDA_CHECK(cudaMemcpyAsync(wav_out + (size_t)b * ld, vs->wav.as<float>() + (size_t)b * Ly_row + vs->c[b],
                                       (size_t)counts[b] * sizeof(float), cudaMemcpyDeviceToDevice, s));
        vs->A[b] += rows[b];
        vs->c[b] = c_new[b];
        if (final_host && final_host[b]) vs->ended[b] = 1;
    }
    CUDA_CHECK(cudaGetLastError());
}

void vocoder_stream_trims(dctts_vocoder_stream vs, int32_t* trim_host) {
    const int B = vs->B;
    for (int b = 0; b < B; ++b)
        REQUIRE(vs->ended[b], "dctts_vocoder_stream_close: utterance " + std::to_string(b) + " has not had its final push, so "
                              "it has no trim");
    VocoderArgs a = vs->args;
    a.wav = vs->wav.as<float>();
    CUDA_CHECK(cudaMemcpyAsync(vs->meta.p, vs->A.data(), B * sizeof(int), cudaMemcpyHostToDevice, vs->s));
    voc_energies(a, vs->s);
    vs->h->launches += 1;
    CUDA_CHECK(cudaGetLastError());
    voc_trims(a, trim_host, vs->s, vs->A.data());
}

}  // namespace

extern "C" {

int dctts_vocoder_stream_open(dctts_handle h, int32_t B, int32_t T_cap, int32_t n_iter, double momentum, void* stream,
                              dctts_vocoder_stream* out) {
    return guarded(h, [&] { vocoder_stream_open(h, B, T_cap, n_iter, momentum, S(h, stream), out); });
}

int dctts_vocoder_stream_push(dctts_vocoder_stream vs, const float* mag, int32_t R, const int32_t* rows_host,
                              const int32_t* final_host, float* wav, int64_t ld, int32_t* counts_host) {
    if (!vs) { g_create_error = "null vocoder stream"; return 1; }
    return guarded(vs->h, [&] { vocoder_stream_push(vs, mag, R, rows_host, final_host, wav, ld, counts_host); });
}

int dctts_vocoder_stream_close(dctts_vocoder_stream vs, int32_t* trim_host) {
    if (!vs) { g_create_error = "null vocoder stream"; return 1; }
    const int rc = guarded(vs->h, [&] {
        if (trim_host) vocoder_stream_trims(vs, trim_host);
        else CUDA_CHECK(cudaStreamSynchronize(vs->s));
    });
    if (rc != 0) cudaStreamSynchronize(vs->s);      // the buffers go now: nothing queued may still use them
    delete vs;
    return rc;
}

int dctts_set_vocoder_params(dctts_handle h, int32_t hop_length, int32_t win_length, float power, float max_db,
                             float ref_db, double preemphasis, int32_t n_iter) {
    return guarded(h, [&] {
        REQUIRE(hop_length >= 1 && win_length >= 1 && n_iter >= 0, "dctts_set_vocoder_params: bad arguments");
        REQUIRE(win_length <= 2 * (h->F - 1), "dctts_set_vocoder_params: win_length " + std::to_string(win_length) +
                                              " exceeds n_fft = " + std::to_string(2 * (h->F - 1)));
        h->voc.hop = hop_length; h->voc.win = win_length; h->voc.power = power; h->voc.max_db = max_db;
        h->voc.ref_db = ref_db; h->voc.preemph = preemphasis; h->voc.n_iter = n_iter;
    });
}

int dctts_spectrogram2wav(dctts_handle h, const float* mag, int32_t B, int32_t T, int32_t n_iter, float* wav,
                          int32_t* trim_host, void* stream) {
    return guarded(h, [&] {
        const char* fn = "dctts_spectrogram2wav";
        REQUIRE(mag && wav, std::string(fn) + ": bad arguments");
        griffin_lim(h, fn, mag, B, T, nullptr, n_iter, 0.0, wav, trim_host, nullptr, S(h, stream));
    });
}

int dctts_spectrogram2wav_ragged(dctts_handle h, const float* mag, int32_t B, int32_t T, const int32_t* lengths_host,
                                 int32_t n_iter, float* wav, int32_t* trim_host, void* stream) {
    return guarded(h, [&] {
        const char* fn = "dctts_spectrogram2wav_ragged";
        REQUIRE(mag && wav && lengths_host, std::string(fn) + ": bad arguments");
        griffin_lim(h, fn, mag, B, T, lengths_host, n_iter, 0.0, wav, trim_host, nullptr, S(h, stream));
    });
}

int dctts_spectrogram2wav_momentum(dctts_handle h, const float* mag, int32_t B, int32_t T, const int32_t* lengths_host,
                                   int32_t n_iter, double momentum, float* wav, int32_t* trim_host, double* convergence,
                                   void* stream) {
    return guarded(h, [&] {
        const char* fn = "dctts_spectrogram2wav_momentum";
        REQUIRE(mag && wav, std::string(fn) + ": bad arguments");
        griffin_lim(h, fn, mag, B, T, lengths_host, n_iter, momentum, wav, trim_host, convergence, S(h, stream));
    });
}

int dctts_vocoder_momentum_step(dctts_handle h, int32_t B, int32_t T, const float* wav, const float* S_in, void* E, void* X,
                                double momentum, float* partials, void* stream) {
    return guarded(h, [&] {
        const std::string fn = "dctts_vocoder_momentum_step";
        REQUIRE(wav && S_in && E && X, fn + ": wav, S, E and X are required");
        const float alpha = momentum_alpha(fn, momentum);
        cudaStream_t s = S(h, stream);
        VocoderArgs a = voc_args(h, fn.c_str(), B, T, s);
        a.wav = const_cast<float*>(wav); a.S = const_cast<float*>(S_in); a.X = static_cast<float2*>(X);
        a.E = static_cast<float2*>(E); a.alpha = alpha; a.part = partials;
        voc_stft_phase(a, s);
        h->launches += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_vocoder_stage(dctts_handle h, int32_t stage, int32_t B, int32_t T, const void* in, const float* S_in, void* out,
                        int32_t* trim_host, void* stream) {
    return guarded(h, [&] {
        const std::string fn = "dctts_vocoder_stage";
        REQUIRE(stage >= 0 && stage <= 4, fn + ": stage " + std::to_string(stage) +
                                          " is not one of 0 prepare, 1 istft, 2 stft_phase, 3 deemph, 4 energies");
        REQUIRE(in && out, fn + ": in and out are required");
        REQUIRE(stage != 2 || S_in, fn + ": stage 2 (stft_phase) needs S (B, T, F)");
        REQUIRE(stage != 3 || in == out, fn + ": stage 3 (deemph) works in place: in must equal out");
        cudaStream_t s = S(h, stream);
        VocoderArgs a = voc_args(h, fn.c_str(), B, T, s);
        static const int launches[5] = {1, 2, 1, 3, 1};
        switch (stage) {
            case 0: a.mag = static_cast<const float*>(in); a.X = static_cast<float2*>(out); voc_prepare(a, s); break;
            case 1: a.X = static_cast<float2*>(const_cast<void*>(in)); a.wav = static_cast<float*>(out); voc_istft(a, s); break;
            case 2:
                a.wav = static_cast<float*>(const_cast<void*>(in)); a.S = const_cast<float*>(S_in); a.X = static_cast<float2*>(out);
                voc_stft_phase(a, s);
                break;
            case 3: a.wav = static_cast<float*>(out); voc_deemph(a, s); break;
            case 4: a.wav = static_cast<float*>(const_cast<void*>(in)); a.mse = static_cast<float*>(out); voc_energies(a, s); break;
        }
        h->launches += launches[stage];
        CUDA_CHECK(cudaGetLastError());
        if (stage == 4) voc_trims(a, trim_host, s);
        else CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_feature_stage(dctts_handle h, int32_t stage, int32_t sample_rate, const void* wav, int32_t dtype, const int64_t* seg_host,
                        int32_t B, int32_t r, int32_t T_b, void* out, void* out2, int32_t* host_out, void* stream) {
    return guarded(h, [&] {
        const std::string fn = "dctts_feature_stage";
        REQUIRE(stage >= 0 && stage <= 2, fn + ": stage " + std::to_string(stage) + " is not one of 0 energies, 1 spectra, 2 tables");
        REQUIRE(out && (out2 || stage == 0) && (host_out || stage == 1) && sample_rate > 0 && B >= 1, fn + ": bad arguments");
        require_fft_size(h, fn);
        cudaStream_t s = S(h, stream);
        if (stage == 2) {
            feat_tables(h, sample_rate, s);
            CUDA_CHECK(cudaMemcpyAsync(out, h->feat_melw.p, (size_t)h->hp.n_mels * h->F * sizeof(float), cudaMemcpyDeviceToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(out2, h->feat_window.p, (size_t)h->voc.win * sizeof(float), cudaMemcpyDeviceToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(host_out, h->feat_range.p, 2 * (size_t)h->hp.n_mels * sizeof(int), cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));
            return;
        }
        REQUIRE(wav && seg_host && (dtype == 0 || dtype == 1), fn + ": wav, its segments and dtype 0 or 1 are required");
        std::vector<FeatSeg> seg(B + 1);
        long long frames = 0;
        for (int b = 0; b < B; ++b) {
            const long long src = stage == 0 ? seg_host[b] : seg_host[2 * b], n = stage == 0 ? seg_host[b + 1] - src : seg_host[2 * b + 1];
            REQUIRE(src >= 0 && n >= 2 && n < (1ll << 30), fn + ": utterance " + std::to_string(b) + " has " + std::to_string(n) +
                                                           " samples (need 2 to 2^30)");
            seg[b] = FeatSeg{src, (int)n, (int)frames};
            const long long T = stage == 0 ? 1 + n / 512 : 1 + n / h->voc.hop;
            REQUIRE(stage == 0 || (r >= 1 && (T + r - 1) / r <= T_b), fn + ": utterance " + std::to_string(b) + " needs " +
                                                                      std::to_string((T + r - 1) / std::max(r, 1)) + " rows at r = " +
                                                                      std::to_string(r) + ", T_b is " + std::to_string(T_b));
            frames += T;
        }
        REQUIRE(frames < (1ll << 31), fn + ": batch too long");
        seg[B] = FeatSeg{0, 0, (int)frames};
        h->feat_seg.ensure(seg.size() * sizeof(FeatSeg));
        FeatSeg* seg_dev = h->feat_seg.as<FeatSeg>();
        CUDA_CHECK(cudaMemcpyAsync(seg_dev, seg.data(), seg.size() * sizeof(FeatSeg), cudaMemcpyHostToDevice, s));
        if (stage == 0) {
            feat_frame_mse(wav, dtype, seg_dev, B, (int)frames, static_cast<float*>(out), s);
            h->launches += 1;
            CUDA_CHECK(cudaGetLastError());
            std::vector<float> mse((size_t)frames);
            CUDA_CHECK(cudaMemcpyAsync(mse.data(), out, mse.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));
            for (int b = 0; b < B; ++b) trim_from_mse(mse.data() + seg[b].f0, 1 + seg[b].len / 512, seg[b].len, host_out + 2 * b);
            return;
        }
        feat_tables(h, sample_rate, s);
        feat_run(feat_args(h, wav, dtype, seg_dev, B, frames, static_cast<float*>(out2), static_cast<float*>(out), T_b, r), s);
        h->launches += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_get_spectrograms(dctts_handle h, const float* wav, int64_t n_samples, int32_t sample_rate, float* mel, float* mag,
                           int32_t t_capacity, int32_t* t_out, int32_t* trim_host, void* stream) {
    return guarded(h, [&] {
        REQUIRE(t_out, "dctts_get_spectrograms: bad arguments");
        const int64_t offsets[2] = {0, n_samples};
        feat_batch(h, "dctts_get_spectrograms", wav, 0, offsets, 1, sample_rate, mel, mag, t_capacity, 1, t_out, trim_host, nullptr,
                   S(h, stream));
    });
}

int dctts_load_spectrograms_batch(dctts_handle h, const void* wav, int32_t dtype, const int64_t* offsets_host, int32_t B,
                                  int32_t sample_rate, float* mel, float* mag, int32_t t_capacity,
                                  int32_t* t_host, int32_t* trim_host, int32_t* T_b_out, void* stream) {
    return guarded(h, [&] {
        feat_batch(h, "dctts_load_spectrograms_batch", wav, dtype, offsets_host, B, sample_rate, mel, mag, t_capacity, h->hp.r,
                   t_host, trim_host, T_b_out, S(h, stream));
    });
}

int dctts_resample_batch(dctts_handle h, const void* wav, int32_t dtype, const int64_t* offsets_host, const int32_t* sr_host,
                         int32_t B, int32_t sr_out, float* out, int64_t out_capacity, int64_t* out_offsets_host, void* stream) {
    return guarded(h, [&] {
        const std::string fn = "dctts_resample_batch";
        REQUIRE(wav && offsets_host && sr_host && out && out_offsets_host && B >= 1 && (dtype == 0 || dtype == 1) && sr_out > 0 &&
                out_capacity >= 0, fn + ": bad arguments");
        std::vector<ResampleUtt> utt(B + 1);
        std::vector<TimeSeg> seg;
        long long total = 0;
        for (int b = 0; b < B; ++b) {
            const std::string who = fn + ": utterance " + std::to_string(b);
            const long long n = offsets_host[b + 1] - offsets_host[b];
            REQUIRE(offsets_host[b] >= 0 && n >= 1 && n < (1ll << 31),
                    who + " has " + std::to_string(n) + " samples (need 1 to 2^31 - 1)");
            REQUIRE(sr_host[b] > 0, who + " has sample rate " + std::to_string(sr_host[b]));
            ResampleUtt& u = utt[b];
            u = ResampleUtt{offsets_host[b], total, n, (int)n, (int)seg.size(), 0, 0, 1.0, 1.0};
            long long n_out = n;
            if (sr_host[b] != sr_out) {                        // resampy.resample (librosa.core.resample, fix=True)
                const double ratio = (double)sr_out / (double)sr_host[b];
                const double x = (double)n * ratio;
                u.n_valid = (long long)x;
                REQUIRE(u.n_valid >= 1, who + ": " + std::to_string(n) + " samples at " + std::to_string(sr_host[b]) +
                                        " Hz are too short to resample to " + std::to_string(sr_out) + " Hz");
                n_out = (long long)std::ceil(x);
                u.ratio = ratio;
                u.scale = std::min(1.0, ratio);
                u.index_step = (int)(u.scale * RS_TABLE);
                REQUIRE(u.index_step >= 1, who + ": sample rate " + std::to_string(sr_host[b]) + " is over 512 times " +
                                           std::to_string(sr_out));
                u.nseg = resample_time_register(u.n_valid, 1.0 / ratio, seg);
            }
            total += n_out;
            REQUIRE(total <= out_capacity, who + " ends at output sample " + std::to_string(total) + ", past out_capacity " +
                                           std::to_string(out_capacity));
        }
        utt[B] = ResampleUtt{0, total, 0, 0, (int)seg.size(), 0, 0, 1.0, 1.0};
        cudaStream_t s = S(h, stream);
        if (!h->rs_win.p) {
            std::vector<double> w;
            resample_filter_table(w);
            h->rs_win.ensure(w.size() * sizeof(double));
            CUDA_CHECK(cudaMemcpyAsync(h->rs_win.p, w.data(), w.size() * sizeof(double), cudaMemcpyHostToDevice, s));
        }
        // one host-to-device copy: B + 1 utterance records, then the time-register segments
        const size_t ub = utt.size() * sizeof(ResampleUtt), sb = seg.size() * sizeof(TimeSeg);
        std::vector<char> tab(ub + sb);
        std::memcpy(tab.data(), utt.data(), ub);
        if (sb) std::memcpy(tab.data() + ub, seg.data(), sb);
        h->rs_tab.ensure(tab.size());
        CUDA_CHECK(cudaMemcpyAsync(h->rs_tab.p, tab.data(), tab.size(), cudaMemcpyHostToDevice, s));
        const ResampleUtt* utt_dev = h->rs_tab.as<ResampleUtt>();
        resample_run(wav, dtype, utt_dev, B, reinterpret_cast<const TimeSeg*>(h->rs_tab.as<char>() + ub), h->rs_win.as<double>(),
                     out, total, s);
        h->launches += 1;
        CUDA_CHECK(cudaGetLastError());
        for (int b = 0; b <= B; ++b) out_offsets_host[b] = utt[b].dst;
    });
}

int32_t dctts_resample_time_register(int64_t n_out, int32_t sr_in, int32_t sr_out, int64_t* t0, double* v0, double* step,
                                     int32_t capacity) {
    if (n_out < 0 || sr_in <= 0 || sr_out <= 0 || capacity < 0) return -1;
    std::vector<TimeSeg> seg;
    const int n = resample_time_register(n_out, 1.0 / ((double)sr_out / (double)sr_in), seg);
    if (n > capacity) return -1;
    for (int i = 0; i < n; ++i) { t0[i] = seg[i].t0; v0[i] = seg[i].v0; step[i] = seg[i].step; }
    return n;
}

}  // extern "C"
