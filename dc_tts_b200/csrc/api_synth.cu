// api_synth.cu -- synthesis: workspace, block runners, chains, attention, the AR decode and the op-level entry points.
// Reference mapping:
//   block semantics ......... modules.py:91-141 (conv1d), :143-197 (hc), :199-247 (conv1d_transpose)
//   graph wiring / shift .... train.py:48-68, :74-77
//   autoregressive loop ..... synthesize.py:45-57
#include "api_internal.cuh"
#include "numerics.cuh"

namespace {

// ---------------------------------------------------------------------------- workspace
// Persistent decode, split-fp16 planes of the recompute's inputs (kernels_decode.cuh: pl_hist, pl_c1), in halfs:
// the input history of every receptive-field block after the first ((DEC_PL_PAD + T) rows per utterance), then one
// DEC_PL_PAD-row stage image per slab of the first block's input for every utterance slot of every cluster.
// `set` (optional) receives the pointers.
size_t decode_plane_halfs(H* h, int B, __half* base = nullptr, DecParams* set = nullptr) {
    const int T = h->hp.max_T;
    const std::vector<int> rows = audiodec_rows(h->audiodec, T);
    size_t off = 0;
    for (size_t i = 1; i < rows.size() && rows[i] > 1; ++i) {
        if (set) set->pl_hist[set->n_enc + i] = base + off;
        off += (size_t)B * h->audiodec[i].cin * 2 * (DEC_PL_PAD + T);
    }
    if (set) { set->pl_c1 = base + off; set->pl_rows = DEC_PL_PAD + T; }
    if (!h->audiodec.empty()) off += (size_t)(B + DEC_GMAX) * h->audiodec[0].cin * 2 * DEC_PL_PAD;
    return off;
}

}  // namespace

// The last persistent decode's per-cluster counters (dec.stats, dec.frames) summed on the host.  Called when they are
// read, and before ensure_ws reallocates their buffers.
void dctts::api::settle_decode_counts(H* h) {
    auto& D = h->dec;
    if (D.last_clusters > 0 && (D.last_moved_frames < 0 || D.frames_pending)) CUDA_CHECK(cudaDeviceSynchronize());
    if (D.last_clusters > 0 && D.last_moved_frames < 0) {
        std::vector<int> st(2 * (size_t)D.last_clusters);
        CUDA_CHECK(cudaMemcpy(st.data(), D.stats.p, st.size() * sizeof(int), cudaMemcpyDeviceToHost));
        D.last_moved_frames = 0; D.last_moved_utt = 0;
        for (int c = 0; c < D.last_clusters; ++c) { D.last_moved_frames += st[2 * c]; D.last_moved_utt += st[2 * c + 1]; }
    }
    if (D.frames_pending) {
        std::vector<int> fr((size_t)D.last_clusters);
        CUDA_CHECK(cudaMemcpy(fr.data(), D.frames.p, fr.size() * sizeof(int), cudaMemcpyDeviceToHost));
        D.last_frames = 0;
        for (int f : fr) D.last_frames += f;
        D.frames_pending = false;
    }
}

// The one place the captured AR step is destroyed; each caller synchronises first as its own ordering needs.
void dctts::api::drop_ar_graph(H* h) {
    if (h->ar_exec) { cudaGraphExecDestroy(h->ar_exec); h->ar_exec = nullptr; h->ar_B = 0; }
}

// Something other than a full-sequence chain wrote the synthesis buffers or the weights: no record describes the last
// call any more.
void dctts::api::chist_clear(H* h, const std::string& why) { h->chist.nets = 0; h->chist.why = why; }

namespace {

// ---------------------------------------------------------------------------- chain history (option chain_history)
// Test aid: with the option on, the full-sequence chains copy each block's rows into handle-owned buffers as they run
// (device to device; no kernel, so the launch sequence is the same with the option off), for dctts_chain_history.
enum { CH_TEXTENC = 0, CH_AUDIOENC = 1, CH_AUDIODEC = 2, CH_SSRN = 3, CH_ATTENTION = 4 };

int chain_net(H* h, const std::vector<LayerDev>& net) {
    if (&net == &h->textenc) return CH_TEXTENC;
    if (&net == &h->audioenc) return CH_AUDIOENC;
    if (&net == &h->audiodec) return CH_AUDIODEC;
    return CH_SSRN;
}

// The start of an entry point whose chains are recorded: the records of earlier calls go stale.
void chist_begin(H* h, const char* who) {
    chist_clear(h, h->opt.chain_history ? std::string("the last call (") + who + ") ran no full-sequence chain of that network"
                                        : std::string("option chain_history was off during the last call (") + who + ")");
}

H::ChainRec& chist_slot(H* h, int net, int slot, int B, int L, int C, int ld, bool planes) {
    auto& v = h->chist.rec[net];
    if ((int)v.size() <= slot) v.resize((size_t)slot + 1);
    H::ChainRec& r = v[(size_t)slot];
    r.B = B; r.L = L; r.C = C; r.ld = ld; r.planes = planes; r.scaled = false;
    h->chist.nets |= 1u << net;
    return r;
}

// slot 0: the first block's input, slot 1 + i: block i's output.  fp32 rows (B * L of them, pitch ld) ...
void chist_f32(Launch& lc, int net, int slot, const float* src, int ld, int B, int L, int C) {
    H* h = lc.h;
    if (!h->opt.chain_history) return;
    H::ChainRec& r = chist_slot(h, net, slot, B, L, C, C, false);
    if (!src) { r.B = 0; return; }                          // the caller did not ask for these rows: nothing kept

    r.a.ensure((size_t)B * L * C * sizeof(float));
    CUDA_CHECK(cudaMemcpy2DAsync(r.a.p, (size_t)C * sizeof(float), src, (size_t)ld * sizeof(float), (size_t)C * sizeof(float),
                                 (size_t)B * L, cudaMemcpyDeviceToDevice, lc.s));
}

// ... or split planes, with the inverse per-utterance scales the first block applies to them (in_inv, or null)
void chist_planes(Launch& lc, int net, int slot, Planes p, int B, int L, int C, const float* in_inv) {
    H* h = lc.h;
    if (!h->opt.chain_history) return;
    H::ChainRec& r = chist_slot(h, net, slot, B, L, C, p.ld, true);
    const size_t bytes = (size_t)B * L * p.ld * sizeof(__half);
    r.a.ensure(bytes); r.b.ensure(bytes);
    CUDA_CHECK(cudaMemcpyAsync(r.a.p, p.hi, bytes, cudaMemcpyDeviceToDevice, lc.s));
    CUDA_CHECK(cudaMemcpyAsync(r.b.p, p.lo, bytes, cudaMemcpyDeviceToDevice, lc.s));
    if (in_inv) {
        r.scaled = true;
        r.inv.ensure((size_t)B * sizeof(float));
        CUDA_CHECK(cudaMemcpyAsync(r.inv.p, in_inv, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, lc.s));
    }
}

// Row pitches of the full-sequence chains' buffers: the pre-LN scratch and the fp32 ping-pong pair (floats), the split
// planes (halfs)
struct ChainLd { size_t scr, act, pl; };
ChainLd chain_ld(H* h) {
    const dctts_hparams& hp = h->hp;
    const int w = std::max(std::max(2 * hp.c, h->F), 2 * hp.d);
    return ChainLd{(size_t)roundup(std::max(std::max(4 * hp.c, h->F), 4 * hp.d), 4), (size_t)roundup(w, 4), (size_t)roundup(w, 8)};
}

void ensure_ws(H* h, int B) {
    if (B <= h->ws_B) return;
    require_no_synth_stream(h, "growing the synthesis workspace");
    chist_clear(h, "the workspace grew after the last chain");
    const dctts_hparams& hp = h->hp;
    const int T = hp.max_T, N = hp.max_N, d = hp.d;
    const size_t rows_ssrn = (size_t)B * T * hp.r;
    // invalidate anything that baked pointers
    if (h->ar_exec) CUDA_CHECK(cudaStreamSynchronize(h->stream));
    drop_ar_graph(h);
    CUDA_CHECK(cudaDeviceSynchronize());
    settle_decode_counts(h);                              // the counter buffers below may move
    h->hist.ok = false;                                   // and so do the buffers dctts_decode_history reads
    const ChainLd ld = chain_ld(h);
    h->scratch.ensure(std::max(rows_ssrn * ld.scr * sizeof(float), (size_t)64 << 20));
    h->act0.ensure(rows_ssrn * ld.act * sizeof(float));
    h->act1.ensure(rows_ssrn * ld.act * sizeof(float));
    h->kv.ensure((size_t)B * N * 2 * d * sizeof(float));
    h->ybuf.ensure((size_t)B * T * hp.n_mels * sizeof(float));
    h->rbuf.ensure((size_t)B * T * 2 * d * sizeof(float));
    h->ad_sig.ensure((size_t)B * T * hp.n_mels * sizeof(float));
    h->ae_out.resize(h->audioenc.size());
    for (size_t i = 0; i < h->audioenc.size(); ++i)
        h->ae_out[i].ensure((size_t)B * T * h->audioenc[i].cout * sizeof(float));
    h->ad_out.resize(h->audiodec.size());
    for (size_t i = 0; i < h->audiodec.size(); ++i)
        h->ad_out[i].ensure((size_t)B * T * h->audiodec[i].cout * sizeof(float));
    h->ibuf.ensure((size_t)(4 + 3 * B + (size_t)B * T) * sizeof(int));
    h->pathbuf.ensure((size_t)(B + 2 * (size_t)B * T) * sizeof(int));
    h->lbuf.ensure((size_t)B * N * sizeof(int));
    for (auto& pb : h->plane) pb.ensure(rows_ssrn * ld.pl * sizeof(__half));
    h->in_inv.ensure((size_t)B * sizeof(float));
    for (int i = 0; i < 10; ++i) {
        const size_t bytes = (size_t)B * T * (i < 2 ? 2 * d : d) * sizeof(__half);
        h->arpl[i].ensure(bytes);
        CUDA_CHECK(cudaMemset(h->arpl[i].p, 0, h->arpl[i].bytes));
    }
    h->dec.scr.ensure((size_t)(B + DEC_GMAX) * 85 * 512 * sizeof(float));
    h->dec.pl.ensure(decode_plane_halfs(h, B) * sizeof(__half));
    CUDA_CHECK(cudaMemset(h->dec.pl.p, 0, h->dec.pl.bytes));     // the DEC_PL_PAD rows in front of t = 0 stay zero
    h->dec.stats.ensure((size_t)2 * B * sizeof(int));
    h->dec.pfinal.ensure((size_t)B * sizeof(int));
    h->dec.frames.ensure((size_t)B * sizeof(int));
    h->ws_B = B;
}

// The buffers a full-sequence chain runs in (pre-LN scratch, the fp32 ping-pong pair, the split-plane pairs) hold r x rows
// of the chain's input, ws_B x max_T as ensure_ws sizes them; SSRN past max_T (long-form synthesis) needs B x T.  Their
// bytes per mel frame of a batch (98688 at the LJ hyperparameters), and what they hold now.
size_t chain_bytes_per_frame(H* h) {
    const ChainLd ld = chain_ld(h);
    return (size_t)h->hp.r * ((ld.scr + 2 * ld.act) * sizeof(float) + 4 * ld.pl * sizeof(__half));
}

size_t chain_ws_bytes(H* h) {
    size_t n = h->scratch.bytes + h->act0.bytes + h->act1.bytes;
    for (auto& pb : h->plane) n += pb.bytes;
    return n;
}

// Grow those buffers in place to B x T frames, as ensure_ws does for a batch: only ever up, the weights and every other
// buffer kept.  The new buffers are allocated before the old ones are freed, so a size that cannot be allocated fails
// the call with the size in its message and leaves the workspace as it was.
void ensure_chain_frames(H* h, int B, int T, const char* who) {
    const dctts_hparams& hp = h->hp;
    const long long rows = (long long)B * T * hp.r;
    REQUIRE(rows < (1ll << 31), std::string(who) + ": B x T = " + std::to_string((long long)B * T) + " frames is " +
                                    std::to_string(rows) + " SSRN rows, more than 2^31 - 1");
    ensure_ws(h, B);
    const ChainLd ld = chain_ld(h);
    const size_t scr = std::max((size_t)rows * ld.scr * sizeof(float), (size_t)64 << 20);
    const size_t act = (size_t)rows * ld.act * sizeof(float), pl = (size_t)rows * ld.pl * sizeof(__half);
    bool grow = h->scratch.bytes < scr || h->act0.bytes < act || h->act1.bytes < act;
    for (auto& pb : h->plane) grow = grow || pb.bytes < pl;
    if (!grow) return;
    require_no_synth_stream(h, who);
    const size_t want = std::max(scr, h->scratch.bytes) + 2 * std::max(act, h->act0.bytes) + 4 * std::max(pl, h->plane[0].bytes);
    DevBuf n_scr, n_act[2], n_pl[4];
    try {
        n_scr.ensure(std::max(scr, h->scratch.bytes));
        for (auto& b : n_act) b.ensure(std::max(act, h->act0.bytes));
        for (int i = 0; i < 4; ++i) n_pl[i].ensure(std::max(pl, h->plane[i].bytes));
    } catch (const std::exception& e) {
        cudaGetLastError();
        throw std::runtime_error(std::string(who) + ": " + std::to_string(B) + " utterances of " + std::to_string(T) +
                                 " frames need a synthesis workspace of " + std::to_string(want) + " bytes (" +
                                 std::to_string(chain_bytes_per_frame(h)) + " bytes per frame), which cannot be allocated: " +
                                 e.what());
    }
    chist_clear(h, "the workspace grew after the last chain");
    drop_ar_graph(h);                                     // the captured AR step has the old pointers baked in
    CUDA_CHECK(cudaDeviceSynchronize());                  // the old buffers are freed with n_* below, unread by then
    std::swap(h->scratch, n_scr); std::swap(h->act0, n_act[0]); std::swap(h->act1, n_act[1]);
    for (int i = 0; i < 4; ++i) std::swap(h->plane[i], n_pl[i]);
}

void ensure_scratch(H* h, size_t bytes);
struct IntBufs { int *j, *p_cur, *p_next, *p_prev, *p_hist; };
IntBufs ints(H* h) {
    int* base = h->ibuf.as<int>();
    IntBufs r;
    r.j = base; r.p_cur = base + 4; r.p_next = r.p_cur + h->ws_B; r.p_prev = r.p_next + h->ws_B;
    r.p_hist = r.p_prev + h->ws_B;
    return r;
}

// ---------------------------------------------------------------------------- block runners

// conv (+bias) into scratch, then the LN / highway epilogue.  `extra_shift` moves every tap
// (AudioEnc's first block reads the mel buffer one frame back: train.py:51).
void run_block(Launch& lc, const LayerDev& l, int rate, bool causal, int act,
               const float* X, int ldx, RowWin win, float* out, int ldo, float* out2, int ldo2,
               int extra_shift = 0) {
    H* h = lc.h;
    REQUIRE(l.kind != K_D, "run_block: transposed conv must use run_deconv");
    ConvArgs c{};
    c.X = X; c.ldx = ldx; c.Y = h->scratch.as<float>(); c.ldy = l.ldw; c.bias = l.bias;
    c.K = l.cin; c.N = l.nconv; c.ldw = l.ldw;
    c.ntaps = l.size;
    const int tot = (l.size - 1) * rate;
    const int left = causal ? tot : tot / 2;
    for (int j = 0; j < l.size; ++j) {
        c.taps[j].W = l.W + (size_t)j * l.cin * l.ldw;
        c.taps[j].shift = j * rate - left + extra_shift;
    }
    c.win = win; c.Lout = win.L; c.ostride = 1; c.ooff = 0;
    LnArgs n{};
    n.Y = c.Y; n.ldy = l.ldw; n.g1 = l.g1; n.b1 = l.b1; n.g2 = l.g2; n.b2 = l.b2;
    n.X = X; n.ldx = ldx; n.out = out; n.ldo = ldo; n.out2 = out2; n.ldo2 = ldo2;
    n.C = l.cout; n.mode = (l.kind == K_HC) ? 1 : 0; n.act = act; n.win = win;
    // option fused_ln (experiment): GEMM and LN epilogue in one launch, the last CTAs of each 16-row block
    // waiting on an arrival counter.  Parity-green but SLOWER than two graph nodes (B=1: 220 vs 187 us per
    // decode step, B=32: 339 vs 303): a kernel boundary inside a CUDA graph costs less than the
    // ticket / spin / L2 round trips that replace it.
    if (h->opt.fused_ln && h->tickets.p && conv_gemm_ln_fusable(c, n)) {
        launch_conv_gemm_ln(c, n, h->tickets.as<int>(), lc.s, h->scratch.bytes); lc.count();
        return;
    }
    GemmOut go = launch_conv_gemm(c, lc.s, h->scratch.bytes); lc.count();
    n.nparts = go.nparts; n.compact = go.compact; n.part_stride = go.part_stride;
    launch_ln_rows(n, lc.s); lc.count();
}

// stride-2 transposed conv (modules.py:232-239): out[2t] = W0 x[t] + W2 x[t-1], out[2t+1] = W1 x[t].
void run_deconv(Launch& lc, const LayerDev& l, const float* X, int ldx, int B, int L, float* out, int ldo) {
    H* h = lc.h;
    ConvArgs c{};
    c.X = X; c.ldx = ldx; c.Y = h->scratch.as<float>(); c.ldy = l.ldw; c.bias = l.bias;
    c.K = l.cin; c.N = l.nconv; c.ldw = l.ldw;
    c.win = RowWin{B, L, L, nullptr}; c.Lout = 2 * L; c.ostride = 2;
    const size_t tapsz = (size_t)l.cin * l.ldw;
    c.ntaps = 2; c.taps[0] = ConvTap{l.W + 0 * tapsz, 0}; c.taps[1] = ConvTap{l.W + 2 * tapsz, -1}; c.ooff = 0;
    launch_conv_gemm(c, lc.s, h->scratch.bytes, false); lc.count();
    c.ntaps = 1; c.taps[0] = ConvTap{l.W + 1 * tapsz, 0}; c.ooff = 1;
    launch_conv_gemm(c, lc.s, h->scratch.bytes, false); lc.count();
    LnArgs n{};
    n.Y = c.Y; n.ldy = l.ldw; n.g1 = l.g1; n.b1 = l.b1; n.out = out; n.ldo = ldo;
    n.C = l.cout; n.mode = 0; n.act = 0; n.win = RowWin{B, 2 * L, 2 * L, nullptr};
    launch_ln_rows(n, lc.s); lc.count();
}

bool chain_tc_ok(H* h, const std::vector<LayerDev>& net);
void run_chain_tc_planes(Launch& lc, const std::vector<LayerDev>& net, Planes cur, int which, int B, int L,
                         float* out, float* out_sig, int first_extra_shift, const float* in_inv, const int* lengths = nullptr,
                         const DevBuf* pl = nullptr);
void run_chain_full_tc(Launch& lc, const std::vector<LayerDev>& net, const float* X, int ldx, int B, int L,
                       float* out, float* out_sig, const int* lengths = nullptr);

// A whole chain over full sequences, ping-ponging act0/act1; the last block writes
// `out` (dense, ld = its cout) and optionally sigmoid(out) into out_sig.
// lengths (device, optional; 1 <= lengths[b] <= L): each utterance's output rows [0, lengths[b] Lout / L) are what the chain
// computes for that utterance alone at L = lengths[b], and its rows past them are zeros.  On the wgmma path that is one
// launch per block over the batch.  The fp32 path's GEMM schedule depends on a launch's row count (split-K below 257 rows,
// tiled above), so one launch over the batch cannot reproduce it: there the lengths are read back and the chain runs once
// per utterance.
void run_chain_full(Launch& lc, const std::vector<LayerDev>& net, const float* X, int ldx, int B, int L,
                    float* out, float* out_sig, const int* lengths = nullptr) {
    H* h = lc.h;
    if (chain_tc_ok(h, net) && (out || out_sig)) { run_chain_full_tc(lc, net, X, ldx, B, L, out, out_sig, lengths); return; }
    if (lengths) {
        std::vector<int> n((size_t)B);
        CUDA_CHECK(cudaMemcpyAsync(n.data(), lengths, n.size() * sizeof(int), cudaMemcpyDeviceToHost, lc.s));
        CUDA_CHECK(cudaStreamSynchronize(lc.s));
        int up = 1;                                        // output rows per input row
        for (auto& l : net) if (l.kind == K_D) up *= 2;
        const int Lout = L * up, C = net.back().cout;
        require_each("ragged chain", "length", n.data(), B, 1, L);
        for (int b = 0; b < B; ++b) {
            const size_t o = (size_t)b * Lout * C, live = (size_t)n[b] * up * C, dead = (size_t)Lout * C - live;
            run_chain_full(lc, net, X + (size_t)b * L * ldx, ldx, 1, n[b], out ? out + o : nullptr, out_sig ? out_sig + o : nullptr);
            if (dead && out) CUDA_CHECK(cudaMemsetAsync(out + o + live, 0, dead * sizeof(float), lc.s));
            if (dead && out_sig) CUDA_CHECK(cudaMemsetAsync(out_sig + o + live, 0, dead * sizeof(float), lc.s));
        }
        chist_clear(h, "the last chain ran once per utterance (per-utterance lengths on the fp32 kernels): its rows are not "
                       "kept as one batch");
        return;
    }
    const int net_id = chain_net(h, net);
    chist_f32(lc, net_id, 0, X, ldx, B, L, net[0].cin);
    const float* cur = X; int ld = ldx; int len = L;
    float* bufs[2] = {h->act0.as<float>(), h->act1.as<float>()};
    int which = 0;
    for (size_t i = 0; i < net.size(); ++i) {
        const LayerDev& l = net[i];
        const bool last = (i + 1 == net.size());
        float* dst = last ? out : bufs[which];
        const int ldo = last ? l.cout : roundup(l.cout, 4);
        if (last && !dst) { dst = bufs[which]; }            // logits not requested: park them
        if (l.kind == K_D) {
            run_deconv(lc, l, cur, ld, B, len, dst, ldo);
            len *= 2;
        } else {
            run_block(lc, l, l.rate, l.causal, l.act, cur, ld, RowWin{B, len, len, nullptr}, dst, ldo,
                      last ? out_sig : nullptr, l.cout);
        }
        chist_f32(lc, net_id, (int)i + 1, dst, ldo, B, len, l.cout);
        cur = dst; ld = ldo; which ^= 1;
    }
}

Planes ws_planes(H* h, int which, int C) {
    Planes p; p.hi = h->plane[2 * which].as<__half>(); p.lo = h->plane[2 * which + 1].as<__half>(); p.ld = roundup(C, 8);
    return p;
}

// One reference block as ONE wgmma kernel (kernels_tc.cu).  X are the split planes of the
// (B, L, cin) input; the output goes to planes and/or fp32 tensors.
void run_block_tc(Launch& lc, const LayerDev& l, int rate, bool causal, int act, Planes X, RowWin win,
                  int TT, int TB, int tiles_t, Planes out, float* out_f32, int ld_f32, float* sig_f32, int ld_sig,
                  Planes sig, int extra_shift = 0, const float* in_inv = nullptr, const int* lengths = nullptr, int len_shift = 0) {
    const LayerDev::TcPack& p = l.tc;
    REQUIRE(p.ok, "tensor-core path not available for this block");
    // the highway residual is read from the input planes unscaled; scaled input planes only reach conv1d blocks
    REQUIRE(!in_inv || p.mode != 1, "hc block with scaled input planes");
    TcArgs a{};
    a.bias = l.bias; a.g1 = l.g1; a.b1 = l.b1; a.g2 = (p.mode == 1) ? l.g2 : l.g1; a.b2 = (p.mode == 1) ? l.b2 : l.b1;
    a.mode = p.mode; a.act = act; a.C = l.cout; a.bn = p.bn; a.half = p.half; a.inv_scale = p.inv_scale; a.in_inv = in_inv;
    const int tiles = ((win.B + TB - 1) / TB) * tiles_t;
    // Option tc_occ2 = 0 (default): the ring holds as many stages as shared memory allows (three for a 256-column hc block,
    // four for a 256-column conv1d, six at 144 columns); 1 gives launches wider than the device a two-stage ring.  The kernel
    // runs one CTA per SM either way.  With one k-block of MMAs in flight the deeper ring is faster: on an H100 SXM (400 W
    // limit) SSRN at B = 32, T = 210 took 13.9 ms per pass against 18.9 ms with two stages.
    H* h = lc.h;
    const bool occ2 = h->opt.tc_occ2 != 0 && !win.jptr && TT == 128 && TB == 1 && tiles * p.ncta >= h->num_sms;
    const int bk = tc_bk();
    a.ntaps = p.ntaps; a.kb_per_tap = p.kb_per_tap * (64 / bk);
    if (p.mode == 2) { a.shifts[0] = 0; a.shifts[1] = -1; }
    else {
        const int tot = (l.size - 1) * rate, left = causal ? tot : tot / 2;
        for (int j = 0; j < l.size; ++j) a.shifts[j] = j * rate - left + extra_shift;
    }
    a.TT = TT; a.TB = TB; a.tiles_t = tiles_t; a.ntiles = tiles; a.win = win;
    a.X = X; a.out = out; a.out_f32 = out_f32; a.ld_f32 = ld_f32; a.sig_f32 = sig_f32; a.ld_sig = ld_sig; a.sig = sig;
    a.lengths = lengths; a.len_shift = len_shift;
    // the A tile is identical in all CTAs of the cluster: fetch it once (TMA multicast) when the
    // tile is 128 consecutive time rows, each CTA contributing 128/ncta of them
    const bool no_mcast = h->opt.tc_mcast == 0;
    a.mcast = (!no_mcast && p.ncta > 1 && TT == 128 && TB == 1) ? 1 : 0;
    const int box_rows = a.mcast ? TT / p.ncta : TT;
    CUtensorMap mAh, mAl;
    tc_make_act_map(&mAh, X.hi, l.cin, X.ld, win.L, win.B, box_rows, TB, bk);
    tc_make_act_map(&mAl, X.lo, l.cin, X.ld, win.L, win.B, box_rows, TB, bk);
    // option tc_debug: progress markers in host-mapped memory, dumped after a synchronising launch
    const bool debug = h->opt.tc_debug != 0;
    static int* dbg_host = nullptr;
    if (debug) {
        if (!dbg_host) CUDA_CHECK(cudaHostAlloc(&dbg_host, 16 * 64 * sizeof(int), cudaHostAllocMapped));
        memset(dbg_host, 0, 16 * 64 * sizeof(int));
        CUDA_CHECK(cudaHostGetDevicePointer(&a.dbg, dbg_host, 0));
    }
    const CUtensorMap mWh = p.mWhi, mWl = p.mWlo;
    // hc on full sequences: the residual tile comes in by TMA and the output planes leave by TMA (staged in the
    // same shared-memory tile), instead of row-scattered 32-byte loads / stores from the epilogue threads
    const bool no_rtma = h->opt.tc_resid_tma == 0;
    CUtensorMap io[4];
    a.resid_tma = 0;
    a.out_tma = 0;
    if (!no_rtma && p.mode == 1 && TT == 128 && TB == 1 && (a.half % 64) == 0) {
        a.resid_tma = 1;
        // TMA stores only on full sequences: in the decode window the tile starts at a negative time coordinate
        // (measured: the launch traps), and there the few output rows are cheap to store directly
        a.out_tma = (out.hi && !win.jptr) ? 1 : 0;
        tc_make_act_map(&io[0], X.hi, l.cin, X.ld, win.L, win.B, 128, 1, 64);
        tc_make_act_map(&io[1], X.lo, l.cin, X.ld, win.L, win.B, 128, 1, 64);
        if (a.out_tma) {
            tc_make_act_map(&io[2], out.hi, l.cout, out.ld, win.L, win.B, 128, 1, 64);
            tc_make_act_map(&io[3], out.lo, l.cout, out.ld, win.L, win.B, 128, 1, 64);
        } else { io[2] = io[0]; io[3] = io[1]; }
    }
    // decode-window launches and launches that fill the machine: two stages (more CTAs in flight on a wide grid,
    // fewer idle bytes on a short reduction); otherwise as many as shared memory holds
    a.stages = std::min((occ2 || win.jptr) ? 2 : tc_stages_for(p.bn, bk, a.resid_tma, a.half), std::max(1, a.ntaps * a.kb_per_tap));
    if (debug)
        fprintf(stderr, "[tc] %s mode=%d ncta=%d bn=%d half=%d stages=%d nkb=%d tiles=%d TT=%d TB=%d L=%d B=%d\n", l.scope.c_str(),
                a.mode, p.ncta, a.bn, a.half, a.stages, a.ntaps * a.kb_per_tap, tiles, TT, TB, win.L, win.B);
    launch_conv_ln_tc(mAh, mAl, mWh, mWl, a.resid_tma ? io : nullptr, a, p.ncta, tiles, bk, lc.s); lc.count();
    if (debug) {
        cudaError_t e = cudaStreamSynchronize(lc.s);
        for (int c = 0; c < std::min(16, p.ncta * tiles); ++c)
            fprintf(stderr, "[tc]  cta %2d: start=%d tmem=0x%x nkb=%d tma=%d mma=%d acc_ready=%d published=%d combined=%d\n", c,
                    dbg_host[64 * c], dbg_host[64 * c + 1], dbg_host[64 * c + 2], dbg_host[64 * c + 3], dbg_host[64 * c + 4],
                    dbg_host[64 * c + 5], dbg_host[64 * c + 6], dbg_host[64 * c + 7]);
        {
            const int* d0 = dbg_host;      // SM-clock deltas of CTA 0
            auto dt = [&](int a_, int b_) { return (d0[b_] - d0[a_]) & 0x7fffffff; };
            fprintf(stderr, "[tc]  cta 0 cycles: setup %d | main loop %d | statistics %d | cluster barrier %d | normalise+stores %d | teardown %d | total %d\n",
                    dt(8, 9), dt(9, 10), dt(10, 11), dt(11, 12), dt(12, 13), dt(13, 14), dt(8, 14));
        }
        if (e != cudaSuccess) throw std::runtime_error(std::string("conv_ln_tc failed: ") + cudaGetErrorString(e));
    }
}

bool chain_tc_ok(H* h, const std::vector<LayerDev>& net) {
    if (h->tensor_path != 1) return false;
    for (auto& l : net) if (!l.tc.ok) return false;
    return true;
}

// Whole chain on the tensor-core path, starting from split planes `cur` (buffer index `which`
// of the ping-pong pair, or -1 for an external buffer): ... -> fp32 out (+ sigmoid).
// in_inv: inverse per-utterance scales of `cur` (launch_f32_to_planes_scaled), or null.  lengths: per-utterance lengths
// at L (device), or null; every block stores its rows past them as zeros (run_chain_full).  pl: four plane buffers to
// ping-pong in instead of the workspace's (a synthesis stream's own), or null; with them no chain history is kept.
void run_chain_tc_planes(Launch& lc, const std::vector<LayerDev>& net, Planes cur, int which, int B, int L,
                         float* out, float* out_sig, int first_extra_shift, const float* in_inv, const int* lengths,
                         const DevBuf* pl) {
    H* h = lc.h;
    int len = L, len_shift = 0;
    int nxt = (which == 0) ? 1 : 0;
    const int net_id = pl ? -1 : chain_net(h, net);
    if (!pl) chist_planes(lc, net_id, 0, cur, B, L, net[0].cin, in_inv);
    for (size_t i = 0; i < net.size(); ++i) {
        const LayerDev& l = net[i];
        const bool last = (i + 1 == net.size());
        Planes dst = last ? Planes{} : pl ? Planes{pl[2 * nxt].as<__half>(), pl[2 * nxt + 1].as<__half>(), roundup(l.cout, 8)}
                                          : ws_planes(h, nxt, l.cout);
        run_block_tc(lc, l, l.rate, l.causal, l.act, cur, RowWin{B, len, len, nullptr}, 128, 1, (len + 127) / 128,
                     dst, last ? out : nullptr, l.cout, last ? out_sig : nullptr, l.cout, Planes{},
                     i == 0 ? first_extra_shift : 0, i == 0 ? in_inv : nullptr, lengths, len_shift);
        if (l.kind == K_D) { len *= 2; ++len_shift; }
        if (pl) {}
        else if (last) chist_f32(lc, net_id, (int)i + 1, out, l.cout, B, len, l.cout);
        else chist_planes(lc, net_id, (int)i + 1, dst, B, len, l.cout, nullptr);
        cur = dst; nxt ^= 1;
    }
}

// The fp32 (B, L, l.cin) input of block l -> its split planes, the way the chains carry that block's input: the first
// block of AudioEnc, AudioDec and SSRN reads audio-level data (mels, R), which silence puts at 1e-8 and below, so its
// planes get a power-of-two scale per utterance (the inverses are returned for the block's epilogue).  Every other
// block reads a LayerNorm output, O(1) per row, or an embedding row, whose magnitude is the committed table's: unscaled
// planes (null).  The op-level entry points follow the same rule, so a network composed block by block computes
// exactly what its chain computes.
// lengths (device, optional, network inputs only): utterance b's rows past lengths[b] are not read and become zero planes.
const float* block_input_planes(Launch& lc, const LayerDev& l, const float* x, int ldx, Planes p, int B, int L,
                                const int* lengths = nullptr) {
    H* h = lc.h;
    const bool net_input = (!h->audioenc.empty() && &l == &h->audioenc[0]) || (!h->audiodec.empty() && &l == &h->audiodec[0]) ||
                           (!h->ssrn.empty() && &l == &h->ssrn[0]);
    if (!net_input) {
        REQUIRE(!lengths, "block_input_planes: per-utterance lengths on a hidden block's input");
        launch_f32_to_planes(x, ldx, p, (long long)B * L, l.cin, lc.s); lc.count();
        return nullptr;
    }
    h->in_inv.ensure((size_t)B * sizeof(float));         // an op-level call may exceed the workspace's batch
    float* in_inv = h->in_inv.as<float>();
    launch_f32_to_planes_scaled(x, ldx, p, B, L, l.cin, in_inv, lc.s, lengths); lc.count();
    return in_inv;
}

// fp32 in -> planes -> chain
void run_chain_full_tc(Launch& lc, const std::vector<LayerDev>& net, const float* X, int ldx, int B, int L,
                       float* out, float* out_sig, const int* lengths) {
    H* h = lc.h;
    Planes cur = ws_planes(h, 0, net[0].cin);
    const float* in_inv = block_input_planes(lc, net[0], X, ldx, cur, B, L, lengths);
    run_chain_tc_planes(lc, net, cur, 0, B, L, out, out_sig, 0, in_inv, lengths);
}

}  // namespace

void dctts::api::run_attention(Launch& lc, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                               RowWin win, int N, const int* pma, float* R, float* align, long long* maxatt,
                               int* p_next, int* p_hist, Planes Rpl) {
    H* h = lc.h;
    REQUIRE(h->hp.d <= 256, "attention: d exceeds 256");
    AttnArgs a{};
    a.Q = Q; a.ldq = ldq; a.K = K; a.ldk = ldk; a.V = V; a.ldv = ldv;
    a.r_hi = Rpl.hi; a.r_lo = Rpl.lo; a.ldr_h = Rpl.ld;
    a.Rout = R; a.ldr = 2 * h->hp.d; a.align = align; a.maxatt = maxatt; a.pma = pma;
    a.p_next = p_next; a.p_hist = p_hist; a.N = N; a.d = h->hp.d; a.win_size = h->hp.attention_win_size;
    a.win = win;
    launch_attention(a, lc.s); lc.count();
}

// Full-sequence attention on the tensor cores (kernels_attn_tc.cu): dense or with the monotonic
// window.  Q, K, V are fp32 device tensors; their split planes are built here.
void dctts::api::run_attention_tc(Launch& lc, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, int B, int T,
                                  int N, const int* pma, float* R, float* align, long long* maxatt, Planes Rpl) {
    H* h = lc.h;
    const int d = h->hp.d, NP = attn_tc_padded_keys(N);
    const size_t need[3] = {(size_t)B * T * d * sizeof(__half), (size_t)B * N * d * sizeof(__half), (size_t)B * d * NP * sizeof(__half)};
    for (int i = 0; i < 6; ++i) h->attpl[i].ensure(need[i / 2]);
    Planes qp, kp, vp;
    qp.hi = h->attpl[0].as<__half>(); qp.lo = h->attpl[1].as<__half>(); qp.ld = d;
    kp.hi = h->attpl[2].as<__half>(); kp.lo = h->attpl[3].as<__half>(); kp.ld = d;
    vp.hi = h->attpl[4].as<__half>(); vp.lo = h->attpl[5].as<__half>(); vp.ld = NP;
    // Q is AudioEnc's last highway output, h1 * LN(.) + (1 - h1) * x: O(1) per row whatever the mels' level, so its planes
    // need no scale (a network input is scaled before AudioEnc's first block instead)
    launch_f32_to_planes(Q, ldq, qp, (long long)B * T, d, lc.s); lc.count();
    launch_attn_kv_planes(K, ldk, V, ldv, kp, vp, B, N, d, lc.s); lc.count();
    AttnTcArgs a{};
    a.Q = Q; a.ldq = ldq; a.R = R; a.ldr = 2 * d; a.Rpl = Rpl; a.align = align; a.maxatt = maxatt; a.pma = pma;
    a.T = T; a.N = N; a.d = d; a.win_size = h->hp.attention_win_size; a.scale = 1.0f / std::sqrt((float)d);
    launch_attention_tc(qp, kp, vp, a, B, lc.s); lc.count();
}

// Receptive-field pyramid of AudioDec for ONE new frame (SURVEY.md App. A / Q1): number of
// trailing rows each block must (re)compute at every AR step.
std::vector<int> dctts::api::audiodec_rows(const std::vector<LayerDev>& net, int T) {
    std::vector<int> rows(net.size(), 1);
    int need = 1;   // rows of this layer's OUTPUT needed
    for (int i = (int)net.size() - 1; i >= 0; --i) {
        rows[i] = std::min(need, T);
        need += (net[i].size - 1) * net[i].rate;    // rows of its input needed
    }
    return rows;
}

namespace {

bool attention_tc_ok(H* h) { return h->tensor_path == 1 && h->hp.d == 256; }

void run_textenc(Launch& lc, const int* L, int B, float* kv_out /* (B,N,2d) */) {
    H* h = lc.h;
    const int N = h->hp.max_N;
    float* emb = h->act1.as<float>();
    // park the embedding at the far end of act1 so the ping-pong (which starts on act0) never
    // overwrites it before the first block has consumed it
    launch_embed(L, h->embed_table, emb, B * N, h->hp.e, lc.s); lc.count();
    // first block reads act1 and writes act0, and so on
    run_chain_full(lc, h->textenc, emb, h->hp.e, B, N, kv_out, nullptr);
}

// Whether AudioDec block i of the graph-per-frame step runs on the tensor cores: at large batches the wide part of the
// pyramid (rows[i] >= 32 of the first four blocks), one 128-row tile per utterance ending at row j.
bool ar_block_on_tc(H* h, int B, size_t i, const std::vector<int>& rows) {
    return h->tensor_path == 1 && B >= 8 && i < 4 && rows[i] >= 32 && h->audiodec[i].tc.ok;
}

// One AR step (synthesize.py:48-54 restated incrementally, exact w.r.t. the reference's
// full recompute): AudioEnc row j, attention over the AudioDec receptive field under the
// CURRENT window, AudioDec pyramid, Y[j] = sigmoid(logits[j]), p <- argmax of row j, j <- j+1.
// `path`: p <- the workspace's window path at j+1 instead, the argmax of row j recorded (h->pathbuf).
void run_ar_step(Launch& lc, int B, bool path) {
    H* h = lc.h;
    const dctts_hparams& hp = h->hp;
    const int T = hp.max_T, N = hp.max_N, d = hp.d;
    IntBufs ib = ints(h);
    // AudioEnc: one new row per utterance; first block reads Y[j-1] (train.py:51)
    const float* cur = h->ybuf.as<float>(); int ld = hp.n_mels;
    for (size_t i = 0; i < h->audioenc.size(); ++i) {
        const LayerDev& l = h->audioenc[i];
        float* dst = h->ae_out[i].as<float>();
        run_block(lc, l, l.rate, l.causal, l.act, cur, ld, RowWin{B, T, 1, ib.j}, dst, l.cout, nullptr, 0,
                  i == 0 ? -1 : 0);
        cur = dst; ld = l.cout;
    }
    const float* Q = cur;
    std::vector<int> rows = audiodec_rows(h->audiodec, T);
    const int att_rows = std::min(T, rows[0] + (h->audiodec[0].size - 1) * h->audiodec[0].rate);
    const float* K = h->kv.as<float>();
    // Large batches run the wide part of the AudioDec pyramid (85..59 rows per utterance) on the
    // tensor cores, one 128-row tile per utterance ending at row j; the narrow tail and the
    // one-row AudioEnc stay on the latency-oriented fp32 kernels.
    auto on_tc = [&](size_t i) { return ar_block_on_tc(h, B, i, rows); };
    auto ar_planes = [&](int idx, int C) {
        Planes p; p.hi = h->arpl[2 * idx].as<__half>(); p.lo = h->arpl[2 * idx + 1].as<__half>(); p.ld = C; return p;
    };
    Planes Rpl = on_tc(0) ? ar_planes(0, 2 * d) : Planes{};
    run_attention(lc, Q, d, K, 2 * d, K + d, 2 * d, RowWin{B, T, att_rows, ib.j}, N, ib.p_cur,
                  h->rbuf.as<float>(), nullptr, nullptr, ib.p_next, ib.p_hist, Rpl);
    cur = h->rbuf.as<float>(); ld = 2 * d;
    Planes cur_pl = Rpl;
    for (size_t i = 0; i < h->audiodec.size(); ++i) {
        const LayerDev& l = h->audiodec[i];
        const bool last = (i + 1 == h->audiodec.size());
        float* dst = h->ad_out[i].as<float>();
        if (on_tc(i)) {
            const bool next_tc = (i + 1 < h->audiodec.size()) && on_tc(i + 1);
            Planes outp = next_tc ? ar_planes((int)i + 1, l.cout) : Planes{};
            run_block_tc(lc, l, l.rate, l.causal, l.act, cur_pl, RowWin{B, T, rows[i], ib.j}, 128, 1, 1, outp,
                         next_tc ? nullptr : dst, l.cout, nullptr, 0, Planes{});
            cur_pl = outp;
        } else {
            run_block(lc, l, l.rate, l.causal, l.act, cur, ld, RowWin{B, T, rows[i], ib.j}, dst, l.cout,
                      last ? h->ybuf.as<float>() : nullptr, hp.n_mels);
        }
        cur = dst; ld = l.cout;
    }
    if (path) {
        int* pb = h->pathbuf.as<int>() + h->ws_B;
        launch_ar_advance_path(ib.p_cur, ib.p_next, ib.j, pb, pb + (size_t)h->ws_B * T, B, T, lc.s);
    } else {
        launch_ar_advance(ib.p_cur, ib.p_next, ib.j, B, lc.s);
    }
    lc.count();
    // keep the window used by this step for the optional final alignment pass
}

void build_ar_graph(H* h, int B, bool path = false) {
    if (h->ar_exec && h->ar_B == B && h->ar_path == path) return;
    drop_ar_graph(h);
    CUDA_CHECK(cudaStreamSynchronize(h->stream));
    cudaGraph_t graph = nullptr;
    int64_t before = h->launches;
    CUDA_CHECK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    try {
        Launch lc{h, h->stream};
        run_ar_step(lc, B, path);
    } catch (...) {
        cudaStreamEndCapture(h->stream, &graph);
        if (graph) cudaGraphDestroy(graph);
        h->launches = before;
        throw;
    }
    CUDA_CHECK(cudaStreamEndCapture(h->stream, &graph));
    h->ar_nodes = h->launches - before;
    h->launches = before;
    cudaError_t e = cudaGraphInstantiate(&h->ar_exec, graph, 0);
    cudaGraphDestroy(graph);
    CUDA_CHECK(e);
    CUDA_CHECK(cudaGetLastError());
    h->ar_B = B;
    h->ar_path = path;
}

// End of utterance for dctts_text2mel_generate_until: device stop positions (B), tail frames, device lengths out (B)
struct Until { const int* stop_pos; int tail; int* lengths; };
// Decode along a window path (dctts_text2mel_generate_path), all in h->pathbuf: lengths (B), path (B, T) padded past
// each length with its last window, the argmax of every frame (B, T)
struct PathRun { const int* lengths; const int* path; int* amax; };
PathRun path_run(H* h) {
    int* pb = h->pathbuf.as<int>();
    return PathRun{pb, pb + h->ws_B, pb + h->ws_B + (size_t)h->ws_B * h->hp.max_T};
}

// Utterances per decode cluster: the fewest that let every cluster be co-resident (a second wave doubles the time).
// reserve (a synthesis stream): the fewest that leave one co-resident cluster slot -- one GPC -- free for the stream's
// SSRN and Griffin-Lim launches, when five per cluster allow it (B <= 5 (max_clusters - 1)); else the usual rule.
int decode_group(const H* h, int B, bool reserve) {
    if (h->opt.decode_group > 0) return h->opt.decode_group;     // measurement override
    int mc = std::max(1, h->dec.max_clusters);
    if (reserve && mc > 1 && (B + DEC_GMAX - 1) / DEC_GMAX <= mc - 1) --mc;
    int G = 1;
    while (G < DEC_GMAX && (B + G - 1) / G > mc) ++G;
    return G;
}

// The whole AR loop as one persistent launch (kernels_decode.cu).  Returns false when this handle / device cannot run it.
// progress (with u; mapped host memory, DEC_PROG_INTS per cluster): run decode_progress_kernel, with decode_group's
// reserving rule.
bool decode_cluster(H* h, int B, int steps, cudaStream_t s, const Until* u, const PathRun* pr = nullptr, int* progress = nullptr) {
    auto& D = h->dec;
    if (!D.ok || h->opt.decode_mode != 1) return false;
    const dctts_hparams& hp = h->hp;
    IntBufs ib = ints(h);
    DecParams P = D.tab;
    for (int li = 0; li < P.nl; ++li) {
        const bool enc = li < P.n_enc;
        P.out_hist[li] = enc ? h->ae_out[li].as<float>() : h->ad_out[li - P.n_enc].as<float>();
        P.in_hist[li] = li == 0 ? nullptr : (li == P.n_enc ? h->rbuf.as<float>() : P.out_hist[li - 1]);
    }
    P.kv = h->kv.as<float>(); P.ybuf = h->ybuf.as<float>(); P.rbuf = h->rbuf.as<float>(); P.pre_scr = D.scr.as<float>();
    decode_plane_halfs(h, h->ws_B, D.pl.as<__half>(), &P);
    P.p_hist = ib.p_hist; P.p_final = D.pfinal.as<int>(); P.stats = D.stats.as<int>();
    P.prof = nullptr;
    P.force_prepass = h->opt.decode_force_prepass != 0;
    P.stop_pos = nullptr; P.lengths = nullptr; P.frames = nullptr; P.tail = 0;
    if (u) {
        // the stream bound is lowered at a frame's attention; the refill cursor must then still be inside that frame
        REQUIRE(P.nch - P.nch_enc >= DEC_NSLOT, "decode: fewer AudioDec weight chunks per frame than ring slots");
        P.stop_pos = u->stop_pos; P.lengths = u->lengths; P.frames = D.frames.as<int>(); P.tail = u->tail;
    } else if (pr) {
        P.lengths = const_cast<int*>(pr->lengths); P.frames = D.frames.as<int>();
    } else if (h->opt.decode_prof) { D.prof.ensure(DEC_NPROF * sizeof(long long)); CUDA_CHECK(cudaMemsetAsync(D.prof.p, 0, DEC_NPROF * sizeof(long long), s)); P.prof = D.prof.as<long long>(); }
    P.B = B;
    P.G = decode_group(h, B, progress != nullptr);
    P.T = hp.max_T; P.N = hp.max_N; P.d = hp.d; P.n_mels = hp.n_mels;
    P.win_size = hp.attention_win_size; P.steps = steps;
    const int n_clusters = (B + P.G - 1) / P.G;
    D.timed = false;
    if (h->opt.decode_timing) {
        for (auto& ev : D.ev) if (!ev) CUDA_CHECK(cudaEventCreate(&ev));
        CUDA_CHECK(cudaEventRecord(D.ev[0], s));
    }
    cudaError_t e = pr ? launch_decode_path(P, pr->path, pr->amax, n_clusters, s)
                  : (u && progress) ? launch_decode_progress(P, progress, n_clusters, s) : launch_decode_cluster(P, n_clusters, s);
    if (e != cudaSuccess) {
        // a device on which the 16-CTA cluster cannot be placed after all: remember it and let the caller take the
        // graph-per-frame loop (another GPU path, not a CPU fallback)
        cudaGetLastError();
        D.ok = false; D.why = std::string("decode_cluster_kernel launch failed: ") + cudaGetErrorString(e);
        return false;
    }
    h->launches += 1;
    if (h->opt.decode_timing) { CUDA_CHECK(cudaEventRecord(D.ev[1], s)); D.timed = true; }
    D.last_clusters = n_clusters; D.last_moved_frames = -1;
    D.frames_pending = u != nullptr || pr != nullptr;
    D.last_frames = D.frames_pending ? -1 : n_clusters * steps;
    return true;
}

// `pr`: the workspace's path (path_run) is already uploaded; the windows follow it
// `progress` (with u): the persistent decode publishes its progress there (decode_cluster); no other loop may run.
void text2mel_generate(H* h, const int* L, int B, int steps, float* Y, int* prev_hist,
                       long long* maxatt, float* align, cudaStream_t s, const Until* u = nullptr, const PathRun* pr = nullptr,
                       int* progress = nullptr) {
    const dctts_hparams& hp = h->hp;
    const int T = hp.max_T, N = hp.max_N, d = hp.d;
    if (steps <= 0 || steps > T) steps = T;
    require_no_synth_stream(h, "the decode");
    ensure_ws(h, B);
    h->hist.ok = false;
    const bool cluster = h->dec.ok && h->opt.decode_mode == 1;
    if (!cluster) build_ar_graph(h, B, pr != nullptr);
    IntBufs ib = ints(h);
    Launch lc{h, s};
    run_textenc(lc, L, B, h->kv.as<float>());
    chist_clear(h, "a decode ran after the last full-sequence chain");
    CUDA_CHECK(cudaMemsetAsync(h->ybuf.p, 0, (size_t)B * T * hp.n_mels * sizeof(float), s));
    CUDA_CHECK(cudaMemsetAsync(h->ibuf.p, 0, (size_t)(4 + 3 * h->ws_B + (size_t)h->ws_B * T) * sizeof(int), s));
    if (pr) CUDA_CHECK(cudaMemcpy2DAsync(ib.p_cur, sizeof(int), pr->path, (size_t)T * sizeof(int), sizeof(int), B,
                                         cudaMemcpyDeviceToDevice, s));   // the window of frame 0
    bool persistent = cluster && decode_cluster(h, B, steps, s, u, pr, progress);
    REQUIRE(persistent || !progress, "the persistent decode is not available: " + h->dec.why);
    if (persistent) {
        // the whole loop ran as one launch
    } else {
        if (cluster) { CUDA_CHECK(cudaStreamSynchronize(s)); build_ar_graph(h, B, pr != nullptr); }
        for (int j = 0; j < steps; ++j) {
            CUDA_CHECK(cudaGraphLaunch(h->ar_exec, s));
            h->launches += h->ar_nodes;
        }
        h->dec.frames_pending = false; h->dec.last_frames = steps;
    }
    if (Y) CUDA_CHECK(cudaMemcpyAsync(Y, h->ybuf.p, (size_t)B * T * hp.n_mels * sizeof(float),
                                      cudaMemcpyDeviceToDevice, s));
    if (prev_hist) CUDA_CHECK(cudaMemcpy2DAsync(prev_hist, (size_t)T * sizeof(int), ib.p_hist,
                                                (size_t)T * sizeof(int), (size_t)T * sizeof(int), B,
                                                cudaMemcpyDeviceToDevice, s));
    if (u) {
        // the persistent kernel wrote the lengths; after the graph-per-frame loop (all frames) they come from the window
        // history by the same rule.  The loop is causal, so rows below a length are those of the full-length run.
        launch_until_finish(u->stop_pos, u->tail, steps, T, hp.n_mels, ib.p_hist, !persistent, u->lengths, Y, prev_hist, B, s);
        lc.count();
    }
    if (maxatt || align) {
        // what the LAST sess.run (j = steps-1) returns: every row under that step's window.
        // p_hist[:, steps-1] is that window; gather it into p_prev.
        CUDA_CHECK(cudaMemcpy2DAsync(ib.p_prev, sizeof(int), ib.p_hist + (steps - 1), (size_t)T * sizeof(int),
                                     sizeof(int), B, cudaMemcpyDeviceToDevice, s));
        const float* K = h->kv.as<float>();
        run_attention(lc, h->ae_out.back().as<float>(), d, K, 2 * d, K + d, 2 * d, RowWin{B, T, T, nullptr}, N,
                      ib.p_prev, h->rbuf.as<float>(), align, maxatt, nullptr, nullptr);
        return;                                            // rbuf now holds the final pass, not the decode's rows
    }
    h->hist.ok = true; h->hist.B = B; h->hist.planes_only = 0;
    if (!persistent) {
        const std::vector<int> rows = audiodec_rows(h->audiodec, T);
        for (size_t i = 0; i + 1 < h->audiodec.size(); ++i)
            if (ar_block_on_tc(h, B, i, rows) && ar_block_on_tc(h, B, i + 1, rows)) h->hist.planes_only |= 1u << i;
    }
}

// The teacher-forced front of the Text2Mel graph over T <= max_T frames: TextEnc at max_N, AudioEnc over the T rows of
// mels (B, T, n_mels) read one frame back (train.py:51), and the attention under the window pma, or dense over all max_N
// keys when pma is null.  R goes to rbuf; on the wgmma path (the return value) its split planes also go to arpl[0..1]
// for AudioDec.  Shared by text2mel_forward and the aligner.
bool text2mel_front(Launch& lc, const int* L, const float* mels, const int* pma, int B, int T, long long* maxatt, float* align) {
    H* h = lc.h;
    require_no_synth_stream(h, "the teacher-forced Text2Mel");
    const dctts_hparams& hp = h->hp;
    const int N = hp.max_N, d = hp.d;
    run_textenc(lc, L, B, h->kv.as<float>());
    const float* K = h->kv.as<float>();
    if (chain_tc_ok(h, h->audioenc) && chain_tc_ok(h, h->audiodec)) {
        // tensor-core path: every block over all B*T rows as one wgmma kernel
        Planes mp = ws_planes(h, 0, hp.n_mels);
        const float* in_inv = block_input_planes(lc, h->audioenc[0], mels, hp.n_mels, mp, B, T);
        float* Q = h->ae_out.back().as<float>();
        run_chain_tc_planes(lc, h->audioenc, mp, 0, B, T, Q, nullptr, -1, in_inv);  // shift: train.py:51
        Planes Rpl; Rpl.hi = h->arpl[0].as<__half>(); Rpl.lo = h->arpl[1].as<__half>(); Rpl.ld = 2 * d;
        if (attention_tc_ok(h))
            run_attention_tc(lc, Q, d, K, 2 * d, K + d, 2 * d, B, T, N, pma, h->rbuf.as<float>(), align, maxatt, Rpl);
        else
            run_attention(lc, Q, d, K, 2 * d, K + d, 2 * d, RowWin{B, T, T, nullptr}, N, pma, h->rbuf.as<float>(),
                          align, maxatt, nullptr, nullptr, Rpl);
        chist_f32(lc, CH_ATTENTION, 1, h->rbuf.as<float>(), 2 * d, B, T, 2 * d);
        return true;
    }
    // AudioEnc over all rows, reading mels shifted by one frame (train.py:51)
    const float* cur = mels; int ld = hp.n_mels;
    chist_f32(lc, CH_AUDIOENC, 0, mels, hp.n_mels, B, T, hp.n_mels);
    for (size_t i = 0; i < h->audioenc.size(); ++i) {
        const LayerDev& l = h->audioenc[i];
        float* dst = h->ae_out[i].as<float>();
        run_block(lc, l, l.rate, l.causal, l.act, cur, ld, RowWin{B, T, T, nullptr}, dst, l.cout, nullptr, 0,
                  i == 0 ? -1 : 0);
        chist_f32(lc, CH_AUDIOENC, (int)i + 1, dst, l.cout, B, T, l.cout);
        cur = dst; ld = l.cout;
    }
    run_attention(lc, cur, d, K, 2 * d, K + d, 2 * d, RowWin{B, T, T, nullptr}, N, pma, h->rbuf.as<float>(),
                  align, maxatt, nullptr, nullptr);
    chist_f32(lc, CH_ATTENTION, 1, h->rbuf.as<float>(), 2 * d, B, T, 2 * d);
    return false;
}

void text2mel_forward(H* h, const int* L, const float* mels, const int* pma, int B, float* Y,
                      long long* maxatt, float* align, cudaStream_t s) {
    const dctts_hparams& hp = h->hp;
    const int T = hp.max_T, d = hp.d;
    chist_begin(h, "dctts_text2mel_forward");
    ensure_ws(h, B);
    h->hist.ok = false;
    Launch lc{h, s};
    if (text2mel_front(lc, L, mels, pma, B, T, maxatt, align)) {
        Planes Rpl; Rpl.hi = h->arpl[0].as<__half>(); Rpl.lo = h->arpl[1].as<__half>(); Rpl.ld = 2 * d;
        run_chain_tc_planes(lc, h->audiodec, Rpl, -1, B, T, h->ad_out.back().as<float>(), Y, 0, nullptr);
        return;
    }
    const float* cur = h->rbuf.as<float>(); int ld = 2 * d;
    chist_f32(lc, CH_AUDIODEC, 0, cur, ld, B, T, ld);
    for (size_t i = 0; i < h->audiodec.size(); ++i) {
        const LayerDev& l = h->audiodec[i];
        const bool last = (i + 1 == h->audiodec.size());
        float* dst = h->ad_out[i].as<float>();
        run_block(lc, l, l.rate, l.causal, l.act, cur, ld, RowWin{B, T, T, nullptr}, dst, l.cout,
                  last ? Y : nullptr, hp.n_mels);
        chist_f32(lc, CH_AUDIODEC, (int)i + 1, dst, l.cout, B, T, l.cout);
        cur = dst; ld = l.cout;
    }
}

// Op-level entry (modules.py signatures): fp32 in, fp32 out, on whichever path is selected.
void run_block_op(Launch& lc, const LayerDev& l, int rate, bool causal, int act, const float* x, int B, int L, float* out) {
    H* h = lc.h;
    chist_clear(h, "an op-level block call ran after the last full-sequence chain");
    const int Lout = (l.kind == K_D) ? 2 * L : L;
    if (h->tensor_path == 1 && l.tc.ok) {
        const size_t need = (size_t)B * L * roundup(l.cin, 8) * sizeof(__half);
        h->plane[0].ensure(need); h->plane[1].ensure(need);
        Planes X = ws_planes(h, 0, l.cin);
        const float* in_inv = block_input_planes(lc, l, x, l.cin, X, B, L);
        run_block_tc(lc, l, rate, causal, act, X, RowWin{B, L, L, nullptr}, 128, 1, (L + 127) / 128, Planes{}, out, l.cout,
                     nullptr, 0, Planes{}, 0, in_inv);
        return;
    }
    ensure_scratch(h, (size_t)B * Lout * l.ldw * sizeof(float));
    if (l.kind == K_D) run_deconv(lc, l, x, l.cin, B, L, out, l.cout);
    else run_block(lc, l, rate, causal, act, x, l.cin, RowWin{B, L, L, nullptr}, out, l.cout, nullptr, 0);
}

LayerDev* find_layer(H* h, const char* scope, int kind) {
    REQUIRE(h->committed, "parameters not committed");
    auto it = h->by_scope.find(scope ? scope : "");
    if (it == h->by_scope.end()) throw std::runtime_error(std::string("unknown scope: ") + (scope ? scope : "(null)"));
    if (it->second->kind != kind) throw std::runtime_error(std::string("scope has a different block kind: ") + scope);
    return it->second;
}

// Grow the pre-LN scratch for an op-level call; a reallocation invalidates the AR graph,
// which has the old pointer baked in.
void ensure_scratch(H* h, size_t bytes) {
    bytes = std::max(bytes, (size_t)64 << 20);     // room for the skinny GEMM's split-K partials
    if (bytes <= h->scratch.bytes) return;
    h->scratch.ensure(bytes);                      // synchronises: no replay of the graph is in flight below
    drop_ar_graph(h);
}

}  // namespace

extern "C" {

int dctts_embed(dctts_handle h, const char* scope, const int32_t* ids, int32_t B, int32_t N, float* out, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        auto it = h->dev_vec.find(std::string(scope ? scope : "") + "/lookup_table");
        REQUIRE(it != h->dev_vec.end(), "dctts_embed: unknown scope");
        chist_clear(h, "an op-level embedding call ran after the last full-sequence chain");
        launch_embed(ids, it->second, out, B * N, h->hp.e, S(h, stream)); h->launches++;
    });
}

int dctts_normalize(dctts_handle h, const char* scope, const float* x, int64_t rows, int32_t C, float* out, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        auto g = h->dev_vec.find(std::string(scope ? scope : "") + "/gamma");
        auto b = h->dev_vec.find(std::string(scope ? scope : "") + "/beta");
        REQUIRE(g != h->dev_vec.end() && b != h->dev_vec.end(), "dctts_normalize: unknown scope");
        REQUIRE(C >= 1 && C <= 1056 && rows < (1ll << 31), "dctts_normalize: unsupported width");
        chist_clear(h, "an op-level LayerNorm call ran after the last full-sequence chain");
        LnArgs n{};
        n.Y = x; n.ldy = C; n.g1 = g->second; n.b1 = b->second; n.out = out; n.ldo = C; n.C = C;
        n.mode = 0; n.act = 0; n.win = RowWin{1, (int)rows, (int)rows, nullptr};
        launch_ln_rows(n, S(h, stream)); h->launches++;
    });
}

int dctts_conv1d(dctts_handle h, const char* scope, const float* x, int32_t B, int32_t L, int32_t rate,
                 int32_t causal, int32_t act, float* out, void* stream) {
    return guarded(h, [&] {
        LayerDev* l = find_layer(h, scope, K_C);
        REQUIRE(B >= 1 && L >= 1 && rate >= 1, "dctts_conv1d: bad sizes");
        Launch lc{h, S(h, stream)};
        run_block_op(lc, *l, rate, causal != 0, act, x, B, L, out);
    });
}

int dctts_hc(dctts_handle h, const char* scope, const float* x, int32_t B, int32_t L, int32_t rate,
             int32_t causal, float* out, void* stream) {
    return guarded(h, [&] {
        LayerDev* l = find_layer(h, scope, K_HC);
        REQUIRE(B >= 1 && L >= 1 && rate >= 1, "dctts_hc: bad sizes");
        Launch lc{h, S(h, stream)};
        run_block_op(lc, *l, rate, causal != 0, 0, x, B, L, out);
    });
}

int dctts_conv1d_transpose(dctts_handle h, const char* scope, const float* x, int32_t B, int32_t L, float* out, void* stream) {
    return guarded(h, [&] {
        LayerDev* l = find_layer(h, scope, K_D);
        REQUIRE(B >= 1 && L >= 1, "dctts_conv1d_transpose: bad sizes");
        Launch lc{h, S(h, stream)};
        run_block_op(lc, *l, 1, false, 0, x, B, L, out);
    });
}

int dctts_textenc(dctts_handle h, const int32_t* L, int32_t B, float* K, float* V, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L && K && V, "dctts_textenc: bad arguments");
        require_no_synth_stream(h, "dctts_textenc");
        chist_begin(h, "dctts_textenc");
        ensure_ws(h, B);
        h->hist.ok = false;
        cudaStream_t s = S(h, stream);
        Launch lc{h, s};
        run_textenc(lc, L, B, h->kv.as<float>());
        const int N = h->hp.max_N, d = h->hp.d;
        const size_t w = (size_t)d * sizeof(float);
        CUDA_CHECK(cudaMemcpy2DAsync(K, w, h->kv.as<float>(), 2 * w, w, (size_t)B * N, cudaMemcpyDeviceToDevice, s));
        CUDA_CHECK(cudaMemcpy2DAsync(V, w, h->kv.as<float>() + d, 2 * w, w, (size_t)B * N, cudaMemcpyDeviceToDevice, s));
    });
}

int dctts_audioenc(dctts_handle h, const float* Sin, int32_t B, int32_t T, float* Q, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && T >= 1 && T <= h->hp.max_T && Sin && Q, "dctts_audioenc: bad arguments (T must be <= max_T)");
        chist_begin(h, "dctts_audioenc");
        ensure_ws(h, B);
        Launch lc{h, S(h, stream)};
        run_chain_full(lc, h->audioenc, Sin, h->hp.n_mels, B, T, Q, nullptr);
    });
}

int dctts_attention(dctts_handle h, const float* Q, const float* K, const float* V, int32_t B, int32_t T, int32_t N,
                    int32_t monotonic, const int32_t* pma, float* R, float* alignments, int64_t* max_attentions,
                    void* stream) {
    return guarded(h, [&] {
        REQUIRE(B >= 1 && T >= 1 && N >= 1 && Q && K && V && R, "dctts_attention: bad arguments");
        REQUIRE(!monotonic || pma, "dctts_attention: monotonic attention needs prev_max_attentions");
        chist_clear(h, "an op-level attention call ran after the last full-sequence chain");
        Launch lc{h, S(h, stream)};
        const int d = h->hp.d;
        if (attention_tc_ok(h))
            run_attention_tc(lc, Q, d, K, d, V, d, B, T, N, monotonic ? pma : nullptr, R, alignments,
                             reinterpret_cast<long long*>(max_attentions), Planes{});
        else
            run_attention(lc, Q, d, K, d, V, d, RowWin{B, T, T, nullptr}, N, monotonic ? pma : nullptr, R, alignments,
                          reinterpret_cast<long long*>(max_attentions), nullptr, nullptr);
    });
}

int dctts_audiodec(dctts_handle h, const float* R, int32_t B, int32_t T, float* Y_logits, float* Y, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && T >= 1 && T <= h->hp.max_T && R && Y, "dctts_audiodec: bad arguments (T must be <= max_T)");
        chist_begin(h, "dctts_audiodec");
        ensure_ws(h, B);
        Launch lc{h, S(h, stream)};
        run_chain_full(lc, h->audiodec, R, 2 * h->hp.d, B, T, Y_logits, Y);
    });
}

int dctts_ssrn(dctts_handle h, const float* Y, int32_t B, int32_t T, float* Z_logits, float* Z, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && T >= 1 && Y && Z, "dctts_ssrn: bad arguments");
        ensure_chain_frames(h, B, T, "dctts_ssrn");
        chist_begin(h, "dctts_ssrn");
        Launch lc{h, S(h, stream)};
        run_chain_full(lc, h->ssrn, Y, h->hp.n_mels, B, T, Z_logits, Z);
    });
}

int dctts_ssrn_ragged(dctts_handle h, const float* Y, int32_t B, int32_t T, const int32_t* lengths, float* Z_logits, float* Z,
                      void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && T >= 1 && Y && Z && lengths, "dctts_ssrn_ragged: bad arguments (lengths non-null)");
        ensure_chain_frames(h, B, T, "dctts_ssrn_ragged");
        chist_begin(h, "dctts_ssrn_ragged");
        Launch lc{h, S(h, stream)};
        run_chain_full(lc, h->ssrn, Y, h->hp.n_mels, B, T, Z_logits, Z, lengths);
    });
}

int dctts_text2mel_forward(dctts_handle h, const int32_t* L, const float* mels, const int32_t* pma, int32_t B,
                           float* Y, int64_t* max_attentions, float* alignments, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L && mels && pma && Y, "dctts_text2mel_forward: bad arguments");
        text2mel_forward(h, L, mels, pma, B, Y, reinterpret_cast<long long*>(max_attentions), alignments, S(h, stream));
    });
}

int dctts_text2mel_generate(dctts_handle h, const int32_t* L, int32_t B, int32_t steps, float* Y, int32_t* prev_hist,
                            int64_t* max_attentions, float* alignments, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L, "dctts_text2mel_generate: bad arguments");
        text2mel_generate(h, L, B, steps, Y, prev_hist, reinterpret_cast<long long*>(max_attentions), alignments,
                          S(h, stream));
    });
}

int dctts_text2mel_generate_until(dctts_handle h, const int32_t* L, int32_t B, int32_t steps, const int32_t* stop_pos,
                                  int32_t tail, float* Y, int32_t* prev_hist, int32_t* lengths, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L && stop_pos && Y && lengths, "dctts_text2mel_generate_until: bad arguments");
        REQUIRE(tail >= 0, "dctts_text2mel_generate_until: tail must be >= 0");
        const Until u{stop_pos, std::min<int>(tail, h->hp.max_T), lengths};
        text2mel_generate(h, L, B, steps, Y, prev_hist, nullptr, nullptr, S(h, stream), &u);
    });
}

namespace {

// `bytes` of host memory to the device at dst, one asynchronous copy on s.  They are staged in the handle's pinned
// buffer, whose only wait is for the previous upload out of it, so the host keeps queueing while earlier work runs.
void upload_host(H* h, void* dst, const void* src, size_t bytes, cudaStream_t s) {
    if (!h->path_uploaded) CUDA_CHECK(cudaEventCreateWithFlags(&h->path_uploaded, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventSynchronize(h->path_uploaded));          // the staging buffer is free again
    if (h->path_pinned_bytes < bytes) {
        if (h->path_pinned) { CUDA_CHECK(cudaFreeHost(h->path_pinned)); h->path_pinned = nullptr; h->path_pinned_bytes = 0; }
        CUDA_CHECK(cudaMallocHost(&h->path_pinned, bytes));
        h->path_pinned_bytes = bytes;
    }
    std::memcpy(h->path_pinned, src, bytes);
    CUDA_CHECK(cudaMemcpyAsync(dst, h->path_pinned, bytes, cudaMemcpyHostToDevice, s));
    CUDA_CHECK(cudaEventRecord(h->path_uploaded, s));
}

// dctts_text2mel_generate_path with the path (B, steps) and the lengths (B) in host memory.  They are checked before
// anything is launched, then uploaded without waiting for the stream (upload_host).
void generate_path(H* h, const int* L, int B, int steps, const int* p, const int* n, float* Y, int* prev_hist,
                   int* argmax_hist, cudaStream_t s) {
    const dctts_hparams& hp = h->hp;
    const int T = hp.max_T;
    const std::string fn = "dctts_text2mel_generate_path";
    require_each(fn, "length", n, B, 1, steps);
    require_each(fn, "window", p, B, 0, hp.max_N - 1, n, steps);
    ensure_ws(h, B);
    const PathRun pr = path_run(h);
    std::vector<int> up((size_t)h->ws_B + (size_t)B * T);      // pathbuf's lengths, then the first B path rows
    std::copy(n, n + B, up.begin());
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < T; ++j)     // past the length: the last window, so no frame there moves it
            up[h->ws_B + (size_t)b * T + j] = p[(size_t)b * steps + std::min(j, n[b] - 1)];
    upload_host(h, const_cast<int*>(pr.lengths), up.data(), up.size() * sizeof(int), s);
    text2mel_generate(h, L, B, steps, Y, prev_hist, nullptr, nullptr, s, nullptr, &pr);
    // rows at and past each length: 0 in Y, -1 in the histories
    int* len = const_cast<int*>(pr.lengths);
    launch_until_finish(nullptr, 0, steps, T, hp.n_mels, nullptr, false, len, Y, prev_hist, B, s);
    if (argmax_hist) {
        CUDA_CHECK(cudaMemcpyAsync(argmax_hist, pr.amax, (size_t)B * T * sizeof(int), cudaMemcpyDeviceToDevice, s));
        launch_until_finish(nullptr, 0, steps, T, hp.n_mels, nullptr, false, len, nullptr, argmax_hist, B, s);
    }
}

// The aligner's host-side checks (lengths n (B), ends e (B), in host memory), made before anything is launched; each
// refusal names the utterance.  Returns the largest end, which sizes the search's shared memory.
int check_align(H* h, const char* who, int B, int N, int T, const int* n, const int* e) {
    const int w = h->hp.attention_win_size;
    REQUIRE(w >= 1 && w <= 256, std::string(who) + ": attention_win_size must be in [1, 256]");
    int smem_max = 0;
    CUDA_CHECK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
    require_each(who, "length", n, B, 1, T);
    for (int b = 0; b < B; ++b)
        REQUIRE(e[b] >= 0, std::string(who) + ": utterance " + std::to_string(b) + " has no EOS (text end " +
                               std::to_string(e[b]) + ")");
    require_each(who, "text end", e, B, 0, N - 1);
    int max_end = 0;
    for (int b = 0; b < B; ++b) {
        const std::string u = std::string(who) + ": utterance " + std::to_string(b);
        if ((long long)e[b] > (long long)(w - 1) * n[b])
            throw std::runtime_error(u + ": its text end " + std::to_string(e[b]) + " cannot be reached in " +
                                     std::to_string(n[b]) + " frames with attention_win_size " + std::to_string(w) +
                                     " (at most (w - 1) * frames): the text is too long for the recording");
        if (2 * ((size_t)e[b] + 1) * sizeof(double) > (size_t)smem_max)
            throw std::runtime_error(u + ": the search's rows for text end " + std::to_string(e[b]) +
                                     " do not fit in the device's " + std::to_string(smem_max) + " bytes of shared memory");
        max_end = std::max(max_end, e[b]);
    }
    return max_end;
}

// The search on A (B, N, T) DEVICE, after check_align: stages the lengths and ends, then one launch for the batch.
void align_search(Launch& lc, const float* A, int B, int N, int T, const int* n, const int* e, int max_end,
                  int* path, int* chars, int* durations, double* score) {
    H* h = lc.h;
    std::vector<int> meta(n, n + B);
    meta.insert(meta.end(), e, e + B);
    h->align.bp.ensure((size_t)B * T * N);
    h->align.meta.ensure(meta.size() * sizeof(int));
    upload_host(h, h->align.meta.p, meta.data(), meta.size() * sizeof(int), lc.s);
    AlignArgs a{};
    a.A = A; a.meta = h->align.meta.as<int>(); a.bp = h->align.bp.as<unsigned char>();
    a.path = path; a.chars = chars; a.durations = durations; a.score = score;
    a.B = B; a.N = N; a.T = T; a.win = h->hp.attention_win_size;
    launch_align_search(a, max_end, lc.s); lc.count();
}

}  // namespace

int dctts_align_search(dctts_handle h, const float* alignments, int32_t B, int32_t N, int32_t T, const int32_t* lengths_host,
                       const int32_t* ends_host, int32_t* path, int32_t* chars, int32_t* durations, double* score,
                       void* stream) {
    return guarded(h, [&] {
        REQUIRE(B >= 1 && N >= 1 && T >= 1 && alignments && lengths_host && ends_host && path && chars && durations && score,
                "dctts_align_search: bad arguments");
        const int max_end = check_align(h, "dctts_align_search", B, N, T, lengths_host, ends_host);
        chist_clear(h, "an alignment search ran after the last full-sequence chain");
        Launch lc{h, S(h, stream)};
        align_search(lc, alignments, B, N, T, lengths_host, ends_host, max_end, path, chars, durations, score);
    });
}

int dctts_text2mel_align(dctts_handle h, const int32_t* L, const float* mels, int32_t B, int32_t T, const int32_t* lengths_host,
                         const int32_t* ends_host, int32_t* path, int32_t* chars, int32_t* durations, double* score,
                         float* alignments, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L && mels && lengths_host && ends_host && path && chars && durations && score,
                "dctts_text2mel_align: bad arguments");
        REQUIRE(T >= 1 && T <= h->hp.max_T, "dctts_text2mel_align: T must be in [1, max_T]");
        const int N = h->hp.max_N;
        const int max_end = check_align(h, "dctts_text2mel_align", B, N, T, lengths_host, ends_host);
        chist_begin(h, "dctts_text2mel_align");
        ensure_ws(h, B);
        h->hist.ok = false;
        Launch lc{h, S(h, stream)};
        float* A = alignments;
        if (!A) {
            h->align.A.ensure((size_t)B * N * T * sizeof(float));
            A = h->align.A.as<float>();
        }
        text2mel_front(lc, L, mels, nullptr, B, T, nullptr, A);
        align_search(lc, A, B, N, T, lengths_host, ends_host, max_end, path, chars, durations, score);
    });
}

int dctts_mcd_dtw(dctts_handle h, const float* X, int32_t Tx, const int32_t* nx_host, const float* Y, int32_t Ty,
                  const int32_t* ny_host, int32_t B, int32_t K, double* mcd, int32_t* pairs, int32_t* path, void* stream) {
    return guarded(h, [&] {
        const int M = h->hp.n_mels;
        REQUIRE(B >= 1 && Tx >= 1 && Ty >= 1 && X && Y && nx_host && ny_host && mcd && pairs, "dctts_mcd_dtw: bad arguments");
        REQUIRE(K >= 1 && K <= M - 1, "dctts_mcd_dtw: K must be in [1, n_mels - 1 = " + std::to_string(M - 1) + "], got " +
                                      std::to_string(K));
        int smem_max = 0;
        CUDA_CHECK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
        // per pair: lengths, back-pointer offset, and the cepstra in shared memory (-1) or at a workspace offset
        const size_t ldc = (size_t)(K | 1);
        std::vector<long long> meta(4 * (size_t)B);
        size_t bp_bytes = 0, cep_doubles = 0, smem = 0;
        require_each("dctts_mcd_dtw", "X length", nx_host, B, 1, Tx);
        require_each("dctts_mcd_dtw", "Y length", ny_host, B, 1, Ty);
        for (int b = 0; b < B; ++b) {
            const std::string u = "dctts_mcd_dtw: utterance " + std::to_string(b);
            const long long nx = nx_host[b], ny = ny_host[b];
            const size_t diag = 3 * (size_t)nx * sizeof(double), cep = (size_t)(nx + ny) * ldc * sizeof(double);
            if (diag > (size_t)smem_max)
                throw std::runtime_error(u + ": three diagonals of " + std::to_string(nx) + " doubles do not fit in the device's " +
                                         std::to_string(smem_max) + " bytes of shared memory");
            const bool staged = diag + cep <= (size_t)smem_max;
            meta[4 * b] = nx; meta[4 * b + 1] = ny; meta[4 * b + 2] = (long long)bp_bytes;
            meta[4 * b + 3] = staged ? -1 : (long long)cep_doubles;
            bp_bytes += (size_t)nx * ny;
            if (!staged) cep_doubles += (size_t)(nx + ny) * ldc;
            smem = std::max(smem, staged ? diag + cep : diag);
        }
        const size_t meta_bytes = meta.size() * sizeof(long long);
        h->mcd.bp.ensure(bp_bytes);
        h->mcd.meta.ensure(meta_bytes);
        h->mcd.cep.ensure(cep_doubles * sizeof(double));
        if (!h->mcd.dct.p) {                                  // D[k, m] = sqrt(2 / M) cos(pi k (2m + 1) / (2M)), k >= 1
            std::vector<double> D((size_t)(M - 1) * M);
            const double pi = 3.141592653589793;
            for (int k = 1; k < M; ++k)
                for (int m = 0; m < M; ++m)
                    D[(size_t)(k - 1) * M + m] = std::sqrt(2.0 / M) * std::cos(pi * k * (2 * m + 1) / (2.0 * M));
            h->mcd.dct.ensure(D.size() * sizeof(double));
            CUDA_CHECK(cudaMemcpy(h->mcd.dct.p, D.data(), D.size() * sizeof(double), cudaMemcpyHostToDevice));
        }
        chist_clear(h, "an MCD-DTW call ran after the last full-sequence chain");
        Launch lc{h, S(h, stream)};
        upload_host(h, h->mcd.meta.p, meta.data(), meta_bytes, lc.s);
        McdArgs a{};
        a.X = X; a.Y = Y; a.meta = h->mcd.meta.as<long long>(); a.dct = h->mcd.dct.as<double>();
        a.cep = h->mcd.cep.as<double>(); a.bp = h->mcd.bp.as<unsigned char>();
        a.mcd = mcd; a.pairs = pairs; a.path = path;
        a.max_db = h->voc.max_db; a.ref_db = h->voc.ref_db;
        a.B = B; a.Tx = Tx; a.Ty = Ty; a.n_mels = M; a.K = K;
        launch_mcd_dtw(a, smem, lc.s); lc.count();
    });
}

int dctts_text2mel_generate_path(dctts_handle h, const int32_t* L, int32_t B, int32_t steps, const int32_t* path,
                                 const int32_t* lengths, float* Y, int32_t* prev_hist, int32_t* argmax_hist, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L && path && lengths && Y, "dctts_text2mel_generate_path: bad arguments");
        REQUIRE(steps >= 1 && steps <= h->hp.max_T, "dctts_text2mel_generate_path: steps must be in [1, max_T]");
        cudaStream_t s = S(h, stream);
        // the path and the lengths are checked on the host: read them back (this waits for the stream)
        std::vector<int> n((size_t)B), p((size_t)B * steps);
        CUDA_CHECK(cudaMemcpyAsync(n.data(), lengths, n.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(p.data(), path, p.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
        generate_path(h, L, B, steps, p.data(), n.data(), Y, prev_hist, argmax_hist, s);
    });
}

int dctts_text2mel_generate_path_host(dctts_handle h, const int32_t* L, int32_t B, int32_t steps, const int32_t* path_host,
                                      const int32_t* lengths_host, float* Y, int32_t* prev_hist, int32_t* argmax_hist,
                                      void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L && path_host && lengths_host && Y, "dctts_text2mel_generate_path_host: bad arguments");
        REQUIRE(steps >= 1 && steps <= h->hp.max_T, "dctts_text2mel_generate_path_host: steps must be in [1, max_T]");
        generate_path(h, L, B, steps, path_host, lengths_host, Y, prev_hist, argmax_hist, S(h, stream));
    });
}

int dctts_synthesize_host(dctts_handle h, const int32_t* L_host, int32_t B, float* Y_host, float* Z_host) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(B >= 1 && L_host && Z_host, "dctts_synthesize_host: bad arguments");
        const dctts_hparams& hp = h->hp;
        const int T = hp.max_T, N = hp.max_N;
        ensure_ws(h, B);
        const size_t zbytes = (size_t)B * T * hp.r * h->F * sizeof(float);
        h->zbuf.ensure(zbytes);
        cudaStream_t s = h->stream;
        CUDA_CHECK(cudaMemcpyAsync(h->lbuf.p, L_host, (size_t)B * N * sizeof(int), cudaMemcpyHostToDevice, s));
        text2mel_generate(h, h->lbuf.as<int>(), B, T, nullptr, nullptr, nullptr, nullptr, s);
        if (Y_host) CUDA_CHECK(cudaMemcpyAsync(Y_host, h->ybuf.p, (size_t)B * T * hp.n_mels * sizeof(float), cudaMemcpyDeviceToHost, s));
        // SSRN in utterance chunks; the device->host copy of chunk i (copy stream) runs under the SSRN of chunk i+1.
        // Z is 3.5 MB per utterance: at PCIe rates the copy of a 32-utterance batch is as long as its SSRN.
        if (!h->copy_stream) {
            CUDA_CHECK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
            for (auto& e : h->chunk_done) CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        }
        // chunk ends: quarters of the batch (B >= 16) with the LAST quarter split again -- only the last chunk's copy is exposed,
        // and a chunk costs the SSRN a partly filled wave (measured ~0.55 ms per extra chunk at B = 32), so more, smaller chunks
        // at the front would cost more than they hide
        int ends[8], nchunk = 0;
        if (B >= 16) { for (int c = 1; c <= 3; ++c) ends[nchunk++] = (int)((long long)B * c / 4); ends[nchunk++] = (int)((long long)B * 7 / 8); ends[nchunk++] = B; }
        else if (B >= 4) { ends[nchunk++] = B / 2; ends[nchunk++] = B; }
        else ends[nchunk++] = B;
        const size_t zrow = (size_t)T * hp.r * h->F;
        Launch lc{h, s};
        int b0 = 0;
        for (int c = 0; c < nchunk; ++c) {
            const int b1 = ends[c];
            if (b1 <= b0) continue;
            float* zc = h->zbuf.as<float>() + (size_t)b0 * zrow;
            run_chain_full(lc, h->ssrn, h->ybuf.as<float>() + (size_t)b0 * T * hp.n_mels, hp.n_mels, b1 - b0, T, nullptr, zc);
            CUDA_CHECK(cudaEventRecord(h->chunk_done[c], s));
            CUDA_CHECK(cudaStreamWaitEvent(h->copy_stream, h->chunk_done[c], 0));
            CUDA_CHECK(cudaMemcpyAsync(Z_host + (size_t)b0 * zrow, zc, (size_t)(b1 - b0) * zrow * sizeof(float),
                                       cudaMemcpyDeviceToHost, h->copy_stream));
            b0 = b1;
        }
        CUDA_CHECK(cudaStreamSynchronize(h->copy_stream));
        CUDA_CHECK(cudaStreamSynchronize(s));
        chist_clear(h, "the last call (dctts_synthesize_host) ran a decode and SSRN in utterance chunks");
    });
}

int dctts_bench_block(dctts_handle h, const char* scope, int32_t B, int32_t L, int32_t iters, int32_t warmup,
                      float* ms_per_kernel, int32_t* n_kernels, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->committed, "parameters not committed");
        REQUIRE(scope && B >= 1 && L >= 1 && iters >= 1 && ms_per_kernel && n_kernels, "dctts_bench_block: bad arguments");
        auto it = h->by_scope.find(scope);
        REQUIRE(it != h->by_scope.end(), "dctts_bench_block: unknown scope");
        const LayerDev& l = *it->second;
        const int Lout = (l.kind == K_D) ? 2 * L : L;
        DevBuf x, y;
        x.ensure((size_t)B * L * l.cin * sizeof(float));
        y.ensure((size_t)B * Lout * l.cout * sizeof(float));
        cudaStream_t s = S(h, stream);
        CUDA_CHECK(cudaMemsetAsync(x.p, 0x3c, x.bytes, s));      // 0x3c3c3c3c = 0.0115 as float
        std::vector<cudaEvent_t> evs;
        std::vector<double> acc;
        int nk = 0;
        for (int i = 0; i < warmup + iters; ++i) {
            Launch lc{h, s};
            evs.clear();
            if (i >= warmup) {
                lc.evs = &evs;
                cudaEvent_t e0; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventRecord(e0, s)); evs.push_back(e0);
            }
            run_block_op(lc, l, l.rate, l.causal, l.act, x.as<float>(), B, L, y.as<float>());
            if (i >= warmup) {
                CUDA_CHECK(cudaStreamSynchronize(s));
                nk = (int)evs.size() - 1;
                if (acc.empty()) acc.assign(nk, 0.0);
                for (int k = 0; k < nk; ++k) {
                    float ms = 0.f;
                    CUDA_CHECK(cudaEventElapsedTime(&ms, evs[k], evs[k + 1]));
                    acc[k] += ms;
                }
                for (auto e : evs) cudaEventDestroy(e);
            }
        }
        REQUIRE(nk <= 8, "dctts_bench_block: too many kernels");
        for (int k = 0; k < nk; ++k) ms_per_kernel[k] = (float)(acc[k] / iters);
        *n_kernels = nk;
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_reserve(dctts_handle h, int32_t max_batch) {
    return guarded(h, [&] {
        REQUIRE(max_batch >= 1, "dctts_reserve: bad batch");
        require_no_synth_stream(h, "dctts_reserve");
        ensure_ws(h, max_batch);
    });
}

int dctts_reserve_frames(dctts_handle h, int32_t B, int32_t T, int64_t* bytes) {
    return guarded(h, [&] {
        REQUIRE(B >= 1 && T >= 1, "dctts_reserve_frames: need B >= 1 and T >= 1, got B = " + std::to_string(B) + ", T = " +
                                      std::to_string(T));
        require_no_synth_stream(h, "dctts_reserve_frames");
        ensure_chain_frames(h, B, T, "dctts_reserve_frames");
        if (bytes) *bytes = (int64_t)chain_ws_bytes(h);
    });
}

int dctts_join_rows(dctts_handle h, const float* Y, int32_t P, int32_t T, const int32_t* piece_len,
                    const int32_t* piece_text_host, const int32_t* piece_pause_host, int32_t K, float silence, int32_t T_out,
                    float* out, int32_t* out_len, void* stream) {
    return guarded(h, [&] {
        const std::string fn = "dctts_join_rows";
        REQUIRE(Y && piece_len && piece_text_host && piece_pause_host && out && out_len, fn + ": bad arguments");
        REQUIRE(P >= 1 && K >= 1 && T >= 1 && T_out >= 1, fn + ": need P, K, T and T_out >= 1, got P = " + std::to_string(P) +
                                                              ", K = " + std::to_string(K) + ", T = " + std::to_string(T) +
                                                              ", T_out = " + std::to_string(T_out));
        std::vector<int> meta(2 * (size_t)P + K + 1);
        int* first = meta.data() + 2 * (size_t)P;
        long long need = 0, rows = 0;                    // the longest text's rows at full-length pieces
        for (int p = 0; p < P; ++p) {
            const int k = piece_text_host[p], pause = piece_pause_host[p];
            REQUIRE(k >= 0 && k < K, fn + ": piece " + std::to_string(p) + " belongs to text " + std::to_string(k) +
                                         ", outside [0, " + std::to_string(K) + ")");
            REQUIRE(p == 0 ? k == 0 : (k == piece_text_host[p - 1] || k == piece_text_host[p - 1] + 1),
                    fn + ": piece " + std::to_string(p) + " belongs to text " + std::to_string(k) +
                        ": each text needs at least one piece, and a text's pieces must follow the previous text's");
            const bool last = p + 1 == P || piece_text_host[p + 1] != k;
            REQUIRE(pause >= 0 && (!last || pause == 0), fn + ": piece " + std::to_string(p) + " has a pause of " +
                                                            std::to_string(pause) + " rows (need >= 0, and 0 after a text's last piece)");
            if (p == 0 || k != piece_text_host[p - 1]) { first[k] = p; rows = 0; }
            rows += (long long)T + pause;
            need = std::max(need, rows);
            meta[p] = k; meta[(size_t)P + p] = pause;
        }
        REQUIRE(piece_text_host[P - 1] == K - 1, fn + ": the pieces cover texts 0 .. " + std::to_string(piece_text_host[P - 1]) +
                                                     ", not all " + std::to_string(K));
        REQUIRE(need <= T_out, fn + ": T_out = " + std::to_string(T_out) + " rows cannot hold a text of full-length pieces (" +
                                   std::to_string(need) + " rows)");
        first[K] = P;
        chist_clear(h, "the long-form join ran after the last full-sequence chain");
        cudaStream_t s = S(h, stream);
        h->join_meta.ensure(meta.size() * sizeof(int));
        upload_host(h, h->join_meta.p, meta.data(), meta.size() * sizeof(int), s);
        JoinArgs a{};
        const int* dm = h->join_meta.as<int>();
        a.Y = Y; a.len = piece_len; a.text = dm; a.pause = dm + P; a.first = dm + 2 * (size_t)P;
        a.out = out; a.out_len = out_len; a.silence = silence;
        a.P = P; a.K = K; a.T = T; a.C = h->hp.n_mels; a.T_out = T_out;
        launch_join_rows(a, s); h->launches++;
    });
}

int dctts_set_tensor_path(dctts_handle h, int32_t mode) {
    return guarded(h, [&] {
        REQUIRE(mode == 0 || mode == 1, "dctts_set_tensor_path: mode must be 0 or 1");
        REQUIRE(!(h->synth_stale && mode == 1), "dctts_set_tensor_path: this handle has been trained -- its packed fp16 weight planes "
                "are stale; load the trained variables (dctts_train_tensor) into a new handle for the wgmma kernel set");
        if (mode != h->tensor_path && h->ar_exec) {      // the captured AR step depends on the mode
            CUDA_CHECK(cudaDeviceSynchronize());
            drop_ar_graph(h);
        }
        h->tensor_path = mode;
    });
}

// Of the last dctts_text2mel_generate on the persistent decode path: frames in which at least one utterance of a cluster
// moved its attention window (summed over clusters), utterance-frames whose receptive field was recomputed, clusters used.
int dctts_decode_stats(dctts_handle h, int32_t* moved_frames, int32_t* moved_utterance_frames, int32_t* clusters) {
    return guarded(h, [&] {
        auto& D = h->dec;
        REQUIRE(D.last_clusters > 0, "dctts_decode_stats: no persistent decode has run on this handle");
        settle_decode_counts(h);
        if (moved_frames) *moved_frames = D.last_moved_frames;
        if (moved_utterance_frames) *moved_utterance_frames = D.last_moved_utt;
        if (clusters) *clusters = D.last_clusters;
    });
}

int dctts_decode_history(dctts_handle h, int32_t what, int32_t layer, void* out, int64_t n, int32_t* joined, void* stream) {
    return guarded(h, [&] {
        REQUIRE(h->hist.ok, "dctts_decode_history: the decode buffers do not hold a generation's state (the last writer was not a "
                            "generation without the final attention pass)");
        const dctts_hparams& hp = h->hp;
        const size_t B = (size_t)h->hist.B, T = hp.max_T, N = hp.max_N, d = hp.d;
        const void* src = nullptr;
        size_t elems = 0;
        int plane = -1;                                   // arpl pair holding the rows instead of an fp32 buffer
        if (what == 0 || what == 1) {
            const auto& net = what == 0 ? h->audioenc : h->audiodec;
            REQUIRE(layer >= 0 && layer < (int)net.size(), "dctts_decode_history: block " + std::to_string(layer) + " outside [0, " +
                                                           std::to_string(net.size()) + ")");
            const auto& buf = what == 0 ? h->ae_out : h->ad_out;
            src = buf[layer].p; elems = B * T * net[layer].cout;
            if (what == 1 && ((h->hist.planes_only >> layer) & 1u)) plane = layer + 1;
        } else if (what == 2) { src = h->rbuf.p; elems = B * T * 2 * d; }
        else if (what == 3) { src = h->kv.p; elems = B * N * 2 * d; }
        else if (what == 4) { src = h->ybuf.p; elems = B * T * hp.n_mels; }
        else if (what == 5) { src = ints(h).p_hist; elems = B * T; }
        else REQUIRE(false, "dctts_decode_history: `what` must be 0..5");
        REQUIRE(out && n == (int64_t)elems, "dctts_decode_history: out must hold " + std::to_string(elems) + " elements");
        cudaStream_t s = S(h, stream);
        if (plane < 0) {
            CUDA_CHECK(cudaMemcpyAsync(out, src, elems * 4, cudaMemcpyDeviceToDevice, s));
        } else {                                          // hi + lo on the host: the aid launches no kernel
            std::vector<__half> hi(elems), lo(elems);
            CUDA_CHECK(cudaMemcpyAsync(hi.data(), h->arpl[2 * plane].p, elems * sizeof(__half), cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaMemcpyAsync(lo.data(), h->arpl[2 * plane + 1].p, elems * sizeof(__half), cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));
            std::vector<float> rows(elems);
            for (size_t i = 0; i < elems; ++i) rows[i] = join_f16(hi[i], lo[i]);
            CUDA_CHECK(cudaMemcpyAsync(out, rows.data(), elems * 4, cudaMemcpyHostToDevice, s));
        }
        CUDA_CHECK(cudaStreamSynchronize(s));
        if (joined) *joined = plane >= 0 ? 1 : 0;
    });
}

namespace {

// The record dctts_chain_history reads, or a refusal naming why there is none.  what: 0 block `layer`'s output, 1 the
// first block's input (layer 0).
const H::ChainRec& chist_find(H* h, const char* who, int net, int layer, int what) {
    static const char* names[5] = {"TextEnc", "AudioEnc", "AudioDec", "SSRN", "the attention"};
    REQUIRE(net >= 0 && net < 5, std::string(who) + ": `net` must be 0..4");
    REQUIRE(what == 0 || what == 1, std::string(who) + ": `what` must be 0 (output) or 1 (input)");
    REQUIRE(what == 0 || layer == 0, std::string(who) + ": only the first block's input is kept");
    REQUIRE((h->chist.nets >> net) & 1u, std::string(who) + ": no rows of " + names[net] + " from the last call: " + h->chist.why);
    const auto& v = h->chist.rec[net];
    const int slot = what == 1 ? 0 : 1 + layer;
    REQUIRE(layer >= 0 && slot < (int)v.size() && v[(size_t)slot].B > 0,
            std::string(who) + ": " + names[net] + " kept no " + (what == 1 ? "input" : "output of block " + std::to_string(layer)) +
            " in the last call");
    return v[(size_t)slot];
}

}  // namespace

int dctts_chain_history_shape(dctts_handle h, int32_t net, int32_t layer, int32_t what, int32_t* B, int32_t* L, int32_t* C) {
    return guarded(h, [&] {
        const H::ChainRec& r = chist_find(h, "dctts_chain_history_shape", net, layer, what);
        if (B) *B = r.B;
        if (L) *L = r.L;
        if (C) *C = r.C;
    });
}

int dctts_chain_history(dctts_handle h, int32_t net, int32_t layer, int32_t what, float* out, int64_t n, int32_t* joined,
                        void* stream) {
    return guarded(h, [&] {
        const H::ChainRec& r = chist_find(h, "dctts_chain_history", net, layer, what);
        const size_t rows = (size_t)r.B * r.L, elems = rows * r.C;
        REQUIRE(out && n == (int64_t)elems, "dctts_chain_history: out must hold " + std::to_string(elems) + " floats");
        cudaStream_t s = S(h, stream);
        if (!r.planes) {
            CUDA_CHECK(cudaMemcpyAsync(out, r.a.p, elems * sizeof(float), cudaMemcpyDeviceToDevice, s));
        } else {                                          // hi + lo (times the utterance's inverse scale) on the host
            const size_t pe = rows * r.ld;
            std::vector<__half> hi(pe), lo(pe);
            std::vector<float> inv((size_t)r.B, 1.f), rows_f(elems);
            CUDA_CHECK(cudaMemcpyAsync(hi.data(), r.a.p, pe * sizeof(__half), cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaMemcpyAsync(lo.data(), r.b.p, pe * sizeof(__half), cudaMemcpyDeviceToHost, s));
            if (r.scaled) CUDA_CHECK(cudaMemcpyAsync(inv.data(), r.inv.p, inv.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));
            for (size_t i = 0; i < rows; ++i)
                for (int c = 0; c < r.C; ++c)
                    rows_f[i * r.C + c] = join_f16(hi[i * r.ld + c], lo[i * r.ld + c]) * inv[i / r.L];
            CUDA_CHECK(cudaMemcpyAsync(out, rows_f.data(), elems * sizeof(float), cudaMemcpyHostToDevice, s));
        }
        CUDA_CHECK(cudaStreamSynchronize(s));
        if (joined) *joined = r.planes ? 1 : 0;
    });
}

// SM-clock lap timers of the last persistent decode run with option decode_prof = 1 (cluster 0, CTA rank 0, thread 0):
// the buckets are listed in include/dctts.h.
int dctts_decode_profile(dctts_handle h, int64_t* cycles, int32_t n) {
    return guarded(h, [&] {
        REQUIRE(cycles && n >= 1 && n <= DEC_NPROF, "dctts_decode_profile: bad arguments");
        REQUIRE(h->dec.prof.p, "dctts_decode_profile: no profiled decode has run (set option decode_prof)");
        CUDA_CHECK(cudaDeviceSynchronize());
        long long v[DEC_NPROF];
        CUDA_CHECK(cudaMemcpy(v, h->dec.prof.p, sizeof(v), cudaMemcpyDeviceToHost));
        for (int i = 0; i < n; ++i) cycles[i] = v[i];
    });
}

}  // extern "C"

// ---------------------------------------------------------------------------- streaming synthesis (DESIGN.md section 8j)
namespace {

// Mel frames of context SSRN needs on each side of a run of committed frames, from the layer table: an output interval at
// the final rate, walked back through the blocks (SAME taps [t - left, t + right]; the transposed conv's output 2t reads
// x[t], x[t - 1] and 2t + 1 reads x[t]).  The walk starts at a whole mel frame, so the result holds for every frame.
void ssrn_halo(const H* h, int& left, int& right) {
    int up = 1;
    for (const LayerDev& l : h->ssrn) if (l.kind == K_D) up *= 2;
    const long long a = 1 << 12, b = a + 1;
    long long lo = a * up, hi = b * up;
    for (int i = (int)h->ssrn.size() - 1; i >= 0; --i) {
        const LayerDev& l = h->ssrn[(size_t)i];
        if (l.kind == K_D) {
            lo = (lo % 2 == 0) ? lo / 2 - 1 : lo / 2;
            hi = (hi - 1) / 2 + 1;
        } else {
            const int tot = (l.size - 1) * l.rate, lft = l.causal ? tot : tot / 2;
            lo -= lft; hi += tot - lft;
        }
    }
    left = (int)(a - lo); right = (int)(hi - b);
}

// The buffers of windowed SSRN: the ping-pong plane pairs, the sigmoid output (W, r L, F), the windows' inverse scales and
// their description (len | utt | row0, `slots` rounds of W each), for up to W windows of L mel frames.
struct SsrnWindows {
    DevBuf pl[4], z, inv, meta;
    int W = 0, L = 0;
};

void ssrn_windows_alloc(H* h, SsrnWindows& sw, int W, int L, int slots) {
    const size_t rows = (size_t)W * L * h->hp.r;
    for (auto& b : sw.pl) b.ensure(rows * chain_ld(h).pl * sizeof(__half));
    sw.z.ensure(rows * h->F * sizeof(float));
    sw.inv.ensure((size_t)W * sizeof(float));
    sw.meta.ensure((size_t)slots * 3 * W * sizeof(int));
    sw.W = W; sw.L = L;
}

// One launch set of windowed SSRN on s: windows `win` (device, len | utt | row0 of W) of Y (B, T, n_mels) -> sw.z, window w's
// rows [0, r len[w]) being what the whole-sequence SSRN gives for those rows of a sequence of len[w] frames, at the fixed
// input scale (launch_mel_windows_to_planes).  L: the longest window.
void ssrn_window_run(H* h, SsrnWindows& sw, const float* Y, int T, const int* win, int W, int L, cudaStream_t s) {
    Launch lc{h, s};
    Planes cur{sw.pl[0].as<__half>(), sw.pl[1].as<__half>(), roundup(h->hp.n_mels, 8)};
    launch_mel_windows_to_planes(Y, T, h->hp.n_mels, win, W, L, cur, sw.inv.as<float>(), s); lc.count();
    run_chain_tc_planes(lc, h->ssrn, cur, 0, W, L, nullptr, sw.z.as<float>(), 0, sw.inv.as<float>(), win, sw.pl);
}

void require_ssrn_windows(H* h, const std::string& fn) {
    REQUIRE(h->committed, fn + ": parameters not committed");
    REQUIRE(chain_tc_ok(h, h->ssrn), fn + ": SSRN has no tensor-core chain on this handle" +
                                         (h->tc16_why.empty() ? std::string() : " (" + h->tc16_why + ")"));
}

}  // namespace

// One synthesis stream: the decode of B utterances publishing its progress, and the SSRN windows and vocoder pushes of
// their chunks on the stream's own side stream.  Host state per utterance: the next chunk, samples committed, done.
struct dctts_synth_stream_s {
    H* h = nullptr;
    cudaStream_t ds = nullptr, ss = nullptr;       // the decode's stream (the caller's), the side stream (owned)
    int B = 0, G = 1, T = 0, chunk = 1, tail = 0, left = 0, right = 0, r = 4, F = 0, slots = 1, Lyw = 0, ldr = 0, rmax = 0;
    int* prog = nullptr;                           // pinned, mapped: DEC_PROG_INTS per cluster
    int* meta_host = nullptr;                      // pinned: the windows of one poll's rounds
    DevBuf stop, len, zfull, push, wavr, wav;
    SsrnWindows sw;
    dctts_vocoder_stream vs = nullptr;
    std::vector<int> next, committed, done, first_frames;

    ~dctts_synth_stream_s() {
        if (ds || ss) { cudaStreamSynchronize(ds); if (ss) cudaStreamSynchronize(ss); }
        if (vs) dctts_vocoder_stream_close(vs, nullptr);
        if (prog) cudaFreeHost(prog);
        if (meta_host) cudaFreeHost(meta_host);
        if (ss) cudaStreamDestroy(ss);
    }
};

namespace {

// What the host knows of utterance b: frames published by its cluster, and its length (-1 while unknown)
struct UttProgress { int frames, len; };
UttProgress utt_progress(const dctts_synth_stream_s* st, int b) {
    const int* p = st->prog + (size_t)(b / st->G) * DEC_PROG_INTS;
    const int f = __atomic_load_n(p, __ATOMIC_ACQUIRE);
    int n = __atomic_load_n(p + 1 + b % st->G, __ATOMIC_RELAXED);
    if (n < 0 && f >= st->T) n = st->T;            // the loop ran every frame without reaching the stop
    return {f, n};
}

// The fixed grid: chunk k of utterance b is mel rows [k chunk, min(len, (k + 1) chunk)), ready once the rows its window
// reads are published.  A chunk that starts at or past a known length does not exist.
bool chunk_ready(const dctts_synth_stream_s* st, int b, UttProgress p) {
    const int a = st->next[b] * st->chunk;
    if (p.len >= 0) return a < p.len && p.frames >= std::min(p.len, a + st->chunk + st->right);
    return p.frames >= a + st->chunk + st->right;
}

// Rounds of one chunk per utterance with a ready one, until none is ready: one SSRN launch set and one vocoder push each.
void synth_rounds(dctts_synth_stream_s* st, const char* fn) {
    H* h = st->h;
    const int B = st->B, r = st->r, F = st->F;
    std::vector<UttProgress> p((size_t)B);
    for (int b = 0; b < B; ++b) p[(size_t)b] = utt_progress(st, b);
    std::vector<int> rows((size_t)B), fin((size_t)B), cnt((size_t)B), a0((size_t)B), e0((size_t)B), s0((size_t)B);
    for (int slot = 0;; ++slot) {
        std::vector<int> ws;
        for (int b = 0; b < B; ++b) if (!st->done[b] && chunk_ready(st, b, p[(size_t)b])) ws.push_back(b);
        std::fill(fin.begin(), fin.end(), 0);
        if (ws.empty()) return;
        REQUIRE(slot < st->slots, std::string(fn) + ": more rounds than chunks per utterance");
        const int W = (int)ws.size();
        int* m = st->meta_host + (size_t)slot * 3 * B;
        int L = 1;
        for (int w = 0; w < W; ++w) {
            const int b = ws[(size_t)w];
            const int n = p[(size_t)b].len >= 0 ? p[(size_t)b].len : st->T;
            const int a = st->next[b] * st->chunk, e = std::min(n, a + st->chunk);
            const int s = std::max(0, a - st->left), t = std::min(n, e + st->right);
            m[w] = t - s; m[W + w] = b; m[2 * W + w] = s;
            a0[(size_t)b] = a; e0[(size_t)b] = e; s0[(size_t)b] = s;
            fin[(size_t)b] = (e == p[(size_t)b].len) ? 1 : 0;
            L = std::max(L, t - s);
        }
        int* md = st->sw.meta.as<int>() + (size_t)slot * 3 * B;
        CUDA_CHECK(cudaMemcpyAsync(md, m, (size_t)3 * W * sizeof(int), cudaMemcpyHostToDevice, st->ss));
        ssrn_window_run(h, st->sw, h->ybuf.as<float>(), st->T, md, W, L, st->ss);
        std::fill(rows.begin(), rows.end(), 0);
        for (int w = 0; w < W; ++w) {
            const int b = ws[(size_t)w];
            const size_t n = (size_t)r * (e0[(size_t)b] - a0[(size_t)b]) * F * sizeof(float);
            const float* src = st->sw.z.as<float>() + ((size_t)w * r * L + (size_t)r * (a0[(size_t)b] - s0[(size_t)b])) * F;
            CUDA_CHECK(cudaMemcpyAsync(st->zfull.as<float>() + ((size_t)b * r * st->T + (size_t)r * a0[(size_t)b]) * F, src, n,
                                       cudaMemcpyDeviceToDevice, st->ss));
            CUDA_CHECK(cudaMemcpyAsync(st->push.as<float>() + (size_t)b * st->rmax * F, src, n, cudaMemcpyDeviceToDevice, st->ss));
            rows[(size_t)b] = r * (e0[(size_t)b] - a0[(size_t)b]);
        }
        if (dctts_vocoder_stream_push(st->vs, st->push.as<float>(), st->rmax, rows.data(), fin.data(), st->wavr.as<float>(),
                                      st->ldr, cnt.data()) != 0)
            throw std::runtime_error(h->err);
        for (int b : ws) {
            if (cnt[(size_t)b] > 0)
                CUDA_CHECK(cudaMemcpyAsync(st->wav.as<float>() + (size_t)b * st->Lyw + st->committed[b],
                                           st->wavr.as<float>() + (size_t)b * st->ldr, (size_t)cnt[(size_t)b] * sizeof(float),
                                           cudaMemcpyDeviceToDevice, st->ss));
            st->committed[b] += cnt[(size_t)b];
            if (st->next[b] == 0) st->first_frames[b] = p[(size_t)b].frames;
            ++st->next[b];
            if (fin[(size_t)b]) st->done[b] = 1;
        }
    }
}

void synth_open(H* h, const int* L, int B, const int* stop_host, int tail, int chunk, int n_iter, double momentum,
                cudaStream_t s, dctts_synth_stream* out) {
    const std::string fn = "dctts_synth_stream_open";
    REQUIRE(out && L && stop_host && B >= 1, fn + ": bad arguments");
    REQUIRE(chunk >= 1, fn + ": chunk must be >= 1 mel frame, got " + std::to_string(chunk));
    REQUIRE(tail >= 0, fn + ": tail must be >= 0");
    REQUIRE(!h->synth, fn + ": a synthesis stream is already open on this handle; close it first");
    REQUIRE(h->committed, fn + ": parameters not committed");
    REQUIRE(h->dec.ok && h->opt.decode_mode == 1,
            fn + ": needs the persistent decode, which this handle cannot run: " +
            (h->dec.ok ? std::string("option decode_mode is 0") : h->dec.why) +
            " (after training, refresh_synthesis() / dctts_refresh_synthesis repacks the weights)");
    require_ssrn_windows(h, fn);
    ensure_ws(h, B);                                  // any growth (and its device synchronisation) before this stream starts
    auto st = std::make_unique<dctts_synth_stream_s>();
    st->h = h; st->ds = s; st->B = B; st->T = h->hp.max_T; st->chunk = std::min(chunk, h->hp.max_T);
    st->tail = std::min(tail, h->hp.max_T); st->r = h->hp.r; st->F = h->F;
    st->G = decode_group(h, B, true);
    ssrn_halo(h, st->left, st->right);
    const int T = st->T, r = st->r, F = st->F, clusters = (B + st->G - 1) / st->G;
    st->slots = (T + st->chunk - 1) / st->chunk;
    st->rmax = r * st->chunk;
    st->Lyw = h->voc.hop * (r * T - 1);
    st->ldr = st->Lyw;
    const int Lw = std::min(T, st->chunk + st->left + st->right);
    CUDA_CHECK(cudaStreamCreateWithFlags(&st->ss, cudaStreamNonBlocking));
    CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&st->prog), (size_t)clusters * DEC_PROG_INTS * sizeof(int), cudaHostAllocMapped));
    for (int c = 0; c < clusters; ++c) {
        st->prog[c * DEC_PROG_INTS] = 0;
        for (int g = 1; g < DEC_PROG_INTS; ++g) st->prog[c * DEC_PROG_INTS + g] = -1;
    }
    CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&st->meta_host), (size_t)st->slots * 3 * B * sizeof(int), cudaHostAllocDefault));
    ssrn_windows_alloc(h, st->sw, B, Lw, st->slots);
    st->stop.ensure((size_t)B * sizeof(int)); st->len.ensure((size_t)B * sizeof(int));
    st->zfull.ensure((size_t)B * r * T * F * sizeof(float));
    st->push.ensure((size_t)B * st->rmax * F * sizeof(float));
    st->wavr.ensure((size_t)B * st->ldr * sizeof(float)); st->wav.ensure((size_t)B * st->Lyw * sizeof(float));
    CUDA_CHECK(cudaMemsetAsync(st->zfull.p, 0, st->zfull.bytes, st->ss));
    if (dctts_vocoder_stream_open(h, B, r * T, n_iter, momentum, st->ss, &st->vs) != 0) throw std::runtime_error(h->err);
    st->next.assign(B, 0); st->committed.assign(B, 0); st->done.assign(B, 0); st->first_frames.assign(B, -1);
    int* prog_dev = nullptr;
    CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&prog_dev), st->prog, 0));
    upload_host(h, st->stop.p, stop_host, (size_t)B * sizeof(int), s);
    const Until u{st->stop.as<int>(), st->tail, st->len.as<int>()};
    text2mel_generate(h, L, B, T, nullptr, nullptr, nullptr, nullptr, s, &u, nullptr, prog_dev);
    h->hist.ok = false;                               // the stream's decode is not kept for dctts_decode_history
    h->synth = st.get();
    *out = st.release();
}

void synth_poll(dctts_synth_stream st, int wait, float* wav, int64_t ld, int32_t* counts, int32_t* done, int32_t* frames) {
    const char* fn = "dctts_synth_stream_poll";
    REQUIRE(counts && done && (wav || ld == 0), std::string(fn) + ": bad arguments");
    REQUIRE(ld >= st->Lyw, std::string(fn) + ": ld must hold a whole utterance, " + std::to_string(st->Lyw) + " samples");
    const int B = st->B;
    auto any_ready = [&] {
        for (int b = 0; b < B; ++b) if (!st->done[b] && chunk_ready(st, b, utt_progress(st, b))) return true;
        return false;
    };
    auto all_done = [&] { return std::all_of(st->done.begin(), st->done.end(), [](int d) { return d != 0; }); };
    while (wait && !all_done() && !any_ready()) {
        const cudaError_t e = cudaStreamQuery(st->ds);
        if (e == cudaErrorNotReady) { cudaGetLastError(); std::this_thread::yield(); continue; }
        CUDA_CHECK(e);                                // a failed decode ends the wait with its error
        REQUIRE(any_ready() || all_done(), std::string(fn) + ": the decode ended without publishing every utterance's frames");
    }
    const std::vector<int> c0 = st->committed;
    synth_rounds(st, fn);
    for (int b = 0; b < B; ++b) {
        counts[b] = st->committed[b] - c0[b];
        if (counts[b] > 0)
            CUDA_CHECK(cudaMemcpyAsync(wav + (size_t)b * ld, st->wav.as<float>() + (size_t)b * st->Lyw + c0[b],
                                       (size_t)counts[b] * sizeof(float), cudaMemcpyDeviceToHost, st->ss));
    }
    CUDA_CHECK(cudaStreamSynchronize(st->ss));
    for (int b = 0; b < B; ++b) {
        done[b] = st->done[b];
        if (frames) frames[b] = utt_progress(st, b).frames;
    }
}

void synth_close(dctts_synth_stream st, int32_t* lengths, int32_t* trim, float* Y, float* Z, int32_t* first_frames) {
    H* h = st->h;
    const int B = st->B, T = st->T;
    CUDA_CHECK(cudaStreamSynchronize(st->ds));
    synth_rounds(st, "dctts_synth_stream_close");     // the decode has ended: every remaining chunk is ready
    if (lengths) CUDA_CHECK(cudaMemcpy(lengths, st->len.p, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost));
    if (first_frames) std::copy(st->first_frames.begin(), st->first_frames.end(), first_frames);
    if (Y) {
        launch_until_finish(st->stop.as<int>(), st->tail, T, T, h->hp.n_mels, nullptr, false, st->len.as<int>(), h->ybuf.as<float>(),
                            nullptr, B, st->ds);
        h->launches += 1;
        CUDA_CHECK(cudaMemcpyAsync(Y, h->ybuf.p, (size_t)B * T * h->hp.n_mels * sizeof(float), cudaMemcpyDeviceToDevice, st->ds));
        CUDA_CHECK(cudaStreamSynchronize(st->ds));
    }
    if (Z) CUDA_CHECK(cudaMemcpyAsync(Z, st->zfull.p, st->zfull.bytes, cudaMemcpyDeviceToDevice, st->ss));
    CUDA_CHECK(cudaStreamSynchronize(st->ss));
    dctts_vocoder_stream vs = st->vs;
    st->vs = nullptr;
    if (dctts_vocoder_stream_close(vs, trim) != 0) throw std::runtime_error(h->err);
}

}  // namespace

void dctts::api::synth_stream_free(dctts_synth_stream_s* st) {
    if (st->h && st->h->synth == st) st->h->synth = nullptr;
    delete st;
}

extern "C" {

int dctts_ssrn_halo(dctts_handle h, int32_t* left, int32_t* right) {
    return guarded(h, [&] {
        REQUIRE(left && right, "dctts_ssrn_halo: bad arguments");
        REQUIRE(h->committed, "dctts_ssrn_halo: parameters not committed");
        int l = 0, r = 0;
        ssrn_halo(h, l, r);
        *left = l; *right = r;
    });
}

int dctts_ssrn_windows(dctts_handle h, const float* Y, int32_t B, int32_t T, const int32_t* starts_host, const int32_t* counts_host,
                       const int32_t* lengths_host, float* Z, int32_t ldz_frames, void* stream) {
    return guarded(h, [&] {
        const std::string fn = "dctts_ssrn_windows";
        REQUIRE(Y && Z && starts_host && counts_host && lengths_host && B >= 1 && T >= 1 && ldz_frames >= 1, fn + ": bad arguments");
        require_ssrn_windows(h, fn);
        require_each(fn, "length", lengths_host, B, 1, T);
        int left = 0, right = 0;
        ssrn_halo(h, left, right);
        std::vector<int> m((size_t)3 * B);
        int L = 1;
        for (int b = 0; b < B; ++b) {
            const int a = starts_host[b], e = a + counts_host[b], n = lengths_host[b];
            REQUIRE(a >= 0 && e > a && e <= n && e - a <= ldz_frames,
                    fn + ": utterance " + std::to_string(b) + " has the window [" + std::to_string(a) + ", " + std::to_string(e) +
                        ") outside its length " + std::to_string(n) + " or past ldz_frames");
            const int s = std::max(0, a - left), t = std::min(n, e + right);
            m[(size_t)b] = t - s; m[(size_t)B + b] = b; m[(size_t)2 * B + b] = s;
            L = std::max(L, t - s);
        }
        cudaStream_t s = S(h, stream);
        SsrnWindows sw;
        ssrn_windows_alloc(h, sw, B, L, 1);
        CUDA_CHECK(cudaMemcpyAsync(sw.meta.p, m.data(), m.size() * sizeof(int), cudaMemcpyHostToDevice, s));
        ssrn_window_run(h, sw, Y, T, sw.meta.as<int>(), B, L, s);
        const int r = h->hp.r, F = h->F;
        for (int b = 0; b < B; ++b)
            CUDA_CHECK(cudaMemcpyAsync(Z + (size_t)b * r * ldz_frames * F,
                                       sw.z.as<float>() + ((size_t)b * r * L + (size_t)r * (starts_host[b] - m[(size_t)2 * B + b])) * F,
                                       (size_t)r * counts_host[b] * F * sizeof(float), cudaMemcpyDeviceToDevice, s));
        CUDA_CHECK(cudaStreamSynchronize(s));         // the window buffers are freed on return
    });
}

int dctts_synth_stream_open(dctts_handle h, const int32_t* L, int32_t B, const int32_t* stop_pos_host, int32_t tail, int32_t chunk,
                            int32_t n_iter, double momentum, void* stream, dctts_synth_stream* out) {
    return guarded(h, [&] { synth_open(h, L, B, stop_pos_host, tail, chunk, n_iter, momentum, S(h, stream), out); });
}

int dctts_synth_stream_poll(dctts_synth_stream ss, int32_t wait, float* wav, int64_t ld, int32_t* counts_host, int32_t* done_host,
                            int32_t* frames_host) {
    if (!ss) { g_create_error = "null synthesis stream"; return 1; }
    return guarded(ss->h, [&] { synth_poll(ss, wait, wav, ld, counts_host, done_host, frames_host); });
}

int dctts_synth_stream_close(dctts_synth_stream ss, int32_t* lengths_host, int32_t* trim_host, float* Y, float* Z,
                             int32_t* first_frames_host) {
    if (!ss) { g_create_error = "null synthesis stream"; return 1; }
    H* h = ss->h;
    const bool outputs = lengths_host || trim_host || Y || Z || first_frames_host;
    const int rc = outputs ? guarded(h, [&] { synth_close(ss, lengths_host, trim_host, Y, Z, first_frames_host); }) : 0;
    synth_stream_free(ss);                            // waits for the decode and the side stream
    return rc;
}

}  // extern "C"
