// api_params.cu -- layer tables; parameter staging and commit; the geometry of the split-fp16 planes and of the persistent
// decode's weight stream, and their packing on the device (kernels_pack.cu).
// Reference mapping: layer tables networks.py:23-68 (TextEnc), :81-124 (AudioEnc), :166-209 (AudioDec), :223-290 (SSRN)
#include "api_internal.cuh"
#include "numerics.cuh"

namespace {

// ---------------------------------------------------------------------------- layer tables
void add_layer(std::vector<LayerDev>& v, const std::string& net, int kind, int idx, int cin, int cout,
               int size, int rate, bool causal, int act) {
    LayerDev l;
    const char* pre = kind == K_C ? "C_" : (kind == K_HC ? "HC_" : "D_");
    l.scope = net + "/" + pre + std::to_string(idx);
    l.kind = kind; l.cin = cin; l.cout = cout; l.size = size; l.rate = rate;
    l.causal = causal; l.act = act;
    l.nconv = (kind == K_HC) ? 2 * cout : cout;
    l.ldw = roundup(l.nconv, 4);
    v.push_back(l);
}

}  // namespace

void dctts::api::build_tables(H* h) {
    const dctts_hparams& hp = h->hp;
    const int d = hp.d, d2 = 2 * hp.d, c = hp.c, F = h->F;
    int i;
    // TextEnc, networks.py:23-68
    {
        auto& v = h->textenc; const std::string n = "Text2Mel/TextEnc"; i = 2;
        add_layer(v, n, K_C, i++, hp.e, d2, 1, 1, false, 1);
        add_layer(v, n, K_C, i++, d2, d2, 1, 1, false, 0);
        for (int rep = 0; rep < 2; ++rep)
            for (int j = 0, r = 1; j < 4; ++j, r *= 3) add_layer(v, n, K_HC, i++, d2, d2, 3, r, false, 0);
        for (int rep = 0; rep < 2; ++rep) add_layer(v, n, K_HC, i++, d2, d2, 3, 1, false, 0);
        for (int rep = 0; rep < 2; ++rep) add_layer(v, n, K_HC, i++, d2, d2, 1, 1, false, 0);
    }
    // AudioEnc, networks.py:81-124
    {
        auto& v = h->audioenc; const std::string n = "Text2Mel/AudioEnc"; i = 1;
        add_layer(v, n, K_C, i++, hp.n_mels, d, 1, 1, true, 1);
        add_layer(v, n, K_C, i++, d, d, 1, 1, true, 1);
        add_layer(v, n, K_C, i++, d, d, 1, 1, true, 0);
        for (int rep = 0; rep < 2; ++rep)
            for (int j = 0, r = 1; j < 4; ++j, r *= 3) add_layer(v, n, K_HC, i++, d, d, 3, r, true, 0);
        for (int rep = 0; rep < 2; ++rep) add_layer(v, n, K_HC, i++, d, d, 3, 3, true, 0);
    }
    // AudioDec, networks.py:166-209
    {
        auto& v = h->audiodec; const std::string n = "Text2Mel/AudioDec"; i = 1;
        add_layer(v, n, K_C, i++, d2, d, 1, 1, true, 0);
        for (int j = 0, r = 1; j < 4; ++j, r *= 3) add_layer(v, n, K_HC, i++, d, d, 3, r, true, 0);
        for (int rep = 0; rep < 2; ++rep) add_layer(v, n, K_HC, i++, d, d, 3, 1, true, 0);
        for (int rep = 0; rep < 3; ++rep) add_layer(v, n, K_C, i++, d, d, 1, 1, true, 1);
        add_layer(v, n, K_C, i++, d, hp.n_mels, 1, 1, true, 0);
    }
    // SSRN, networks.py:223-290
    {
        auto& v = h->ssrn; const std::string n = "SSRN"; i = 1;
        add_layer(v, n, K_C, i++, hp.n_mels, c, 1, 1, false, 0);
        for (int j = 0, r = 1; j < 2; ++j, r *= 3) add_layer(v, n, K_HC, i++, c, c, 3, r, false, 0);
        for (int rep = 0; rep < 2; ++rep) {
            add_layer(v, n, K_D, i++, c, c, 3, 1, false, 0);
            for (int j = 0, r = 1; j < 2; ++j, r *= 3) add_layer(v, n, K_HC, i++, c, c, 3, r, false, 0);
        }
        add_layer(v, n, K_C, i++, c, 2 * c, 1, 1, false, 0);
        for (int rep = 0; rep < 2; ++rep) add_layer(v, n, K_HC, i++, 2 * c, 2 * c, 3, 1, false, 0);
        add_layer(v, n, K_C, i++, 2 * c, F, 1, 1, false, 0);
        for (int rep = 0; rep < 2; ++rep) add_layer(v, n, K_C, i++, F, F, 1, 1, false, 1);
        add_layer(v, n, K_C, i, F, F, 1, 1, false, 0);     // networks.py:285-290 (counter not advanced)
    }
    for (auto* vec : {&h->textenc, &h->audioenc, &h->audiodec, &h->ssrn})
        for (auto& l : *vec) h->by_scope[l.scope] = &l;
}

namespace {

// ---------------------------------------------------------------------------- parameters
const HostParam& need(H* h, const std::string& name, std::vector<int64_t> shape) {
    auto it = h->staged.find(name);
    if (it == h->staged.end()) throw std::runtime_error("missing variable: " + name);
    if (it->second.shape != shape) throw std::runtime_error("bad shape for variable: " + name);
    return it->second;
}

template <class T> T* upload(H* h, const std::vector<T>& v) {
    DevBuf& b = h->param_bufs.emplace_back();
    b.ensure(v.size() * sizeof(T));
    CUDA_CHECK(cudaMemcpy(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return b.as<T>();
}

float* upload_vec(H* h, const std::string& name, int n, int padded) {
    const HostParam& p = need(h, name, {n});
    std::vector<float> v(padded, 0.f);
    std::copy(p.data.begin(), p.data.end(), v.begin());
    float* d = upload(h, v);
    h->dev_vec[name] = d;
    h->n_params += n;
    return d;
}

// Split-fp16 planes for the wgmma kernel (kernels_tc.cu): the geometry, the two planes and their tensor maps.  Rows are
// accumulator columns in cluster-slice order (CTA i owns rows [i*bn, (i+1)*bn); for hc / transposed conv its first
// `half` rows are the first LN half, the rest the second), columns are k = tap*cin_pad + ci.  pack_weights fills them
// with the weights multiplied by weight_scale (numerics.cuh); the kernel multiplies the accumulator back.
void tc_tables(H* h, LayerDev& l) {
    LayerDev::TcPack& p = l.tc;
    const int cin_pad = roundup(l.cin, 64);
    p.kb_per_tap = cin_pad / 64;
    if (l.kind == K_C) {
        p.mode = 0; p.ntaps = l.size;
        // small nets (<= 256 channels) are used on few rows (decode): prefer more, narrower CTAs
        const int maxbn = (l.cout <= 256 && l.cout % 64 == 0) ? 64 : 256;
        p.ncta = 1;
        while (roundup((l.cout + p.ncta - 1) / p.ncta, 16) > maxbn) p.ncta *= 2;
        p.bn = roundup((l.cout + p.ncta - 1) / p.ncta, 16); p.half = p.bn;
    } else {
        p.mode = (l.kind == K_HC) ? 1 : 2; p.ntaps = (l.kind == K_HC) ? l.size : 2;
        p.half = (l.cout <= 256) ? 32 : 128; p.bn = 2 * p.half; p.ncta = l.cout / p.half;   // decode nets: 8 narrow CTAs per tile
        if (l.cout % p.half) return;
    }
    if (p.ncta > 8) {
        // the F = 2049 conv1d blocks: a 16-CTA cluster of the 144-column kernel, if one can be co-resident on this device
        if (p.mode != 0 || p.ncta > 16 || p.bn != 144) return;
        if (h->tc16_clusters < 0) {
            h->tc16_clusters = conv_ln_tc_max_clusters(16, 144, tc_bk());
            if (h->tc16_clusters < 1) h->tc16_why = "a 16-CTA cluster of the 144-column block kernel cannot be scheduled on this device";
        }
        if (h->tc16_clusters < 1) return;
    }
    p.Ktot = p.ntaps * cin_pad; p.nrows = p.ncta * p.bn;
    const size_t bytes = (size_t)p.nrows * p.Ktot * sizeof(__half);
    DevBuf& hi = h->param_bufs.emplace_back();
    DevBuf& lo = h->param_bufs.emplace_back();
    hi.ensure(bytes); lo.ensure(bytes);
    p.Whi = hi.as<__half>(); p.Wlo = lo.as<__half>();
    tc_make_w_map(&p.mWhi, p.Whi, p.Ktot, p.nrows, p.bn, tc_bk());
    tc_make_w_map(&p.mWlo, p.Wlo, p.Ktot, p.nrows, p.bn, tc_bk());
    p.ok = true;
}

void commit_layer(H* h, LayerDev& l) {
    const int k = l.size, cin = l.cin, nconv = l.nconv, ldw = l.ldw;
    std::vector<float> W((size_t)k * cin * ldw, 0.f);
    if (l.kind == K_D) {
        // TF kernel [1, k, Cout, Cin] (modules.py:232-239) -> [tap][Cin][ldw]
        const HostParam& p = need(h, l.scope + "/conv2d_transpose/kernel", {1, k, l.cout, cin});
        for (int j = 0; j < k; ++j)
            for (int co = 0; co < l.cout; ++co)
                for (int ci = 0; ci < cin; ++ci)
                    W[((size_t)j * cin + ci) * ldw + co] = p.data[((size_t)j * l.cout + co) * cin + ci];
        l.bias = upload_vec(h, l.scope + "/conv2d_transpose/bias", l.cout, ldw);
        h->n_params += (int64_t)k * l.cout * cin;
    } else {
        // TF kernel [k, Cin, Nconv] (modules.py:134,187) -> same order, rows padded to ldw
        const HostParam& p = need(h, l.scope + "/conv1d/kernel", {k, cin, nconv});
        for (size_t row = 0; row < (size_t)k * cin; ++row)
            std::copy(p.data.begin() + row * nconv, p.data.begin() + (row + 1) * nconv, W.begin() + row * ldw);
        l.bias = upload_vec(h, l.scope + "/conv1d/bias", nconv, ldw);
        h->n_params += (int64_t)k * cin * nconv;
    }
    l.W = upload(h, W);
    tc_tables(h, l);
    if (l.kind == K_HC) {
        l.g1 = upload_vec(h, l.scope + "/H1/gamma", l.cout, l.cout);
        l.b1 = upload_vec(h, l.scope + "/H1/beta", l.cout, l.cout);
        l.g2 = upload_vec(h, l.scope + "/H2/gamma", l.cout, l.cout);
        l.b2 = upload_vec(h, l.scope + "/H2/beta", l.cout, l.cout);
    } else {
        l.g1 = upload_vec(h, l.scope + "/normalize/gamma", l.cout, l.cout);
        l.b1 = upload_vec(h, l.scope + "/normalize/beta", l.cout, l.cout);
    }
}

// ---------------------------------------------------------------------------- persistent decode tables
// Layer / chunk tables and the per-rank weight streams of the cluster decode kernel (kernels_decode.cu).
// Stream of rank r = for every block of AudioEnc then AudioDec, for every tap, for every chunk of <= 4096 floats:
// the block's weight columns owned by rank r ([k/4][column][4]).  hc blocks: columns [0, cs) are the gate
// channels r*cs.., [cs, 2cs) the info channels of the same index (modules.py:188-193); conv blocks: cs columns
// (+ zero columns up to a multiple of 4).  The tables depend on the shapes only; pack_weights writes the stream.
void decode_tables(H* h) {
    auto& D = h->dec;
    D.ok = false; D.tables_ok = false;
    const dctts_hparams& hp = h->hp;
    const int d = hp.d;
    if (d != 256) { D.why = "persistent decode needs d = 256"; return; }
    if (hp.n_mels % DEC_NC || hp.n_mels > 128 || hp.attention_win_size > 4 || hp.attention_win_size < 1) { D.why = "persistent decode: unsupported n_mels / window"; return; }
    std::vector<LayerDev*> nets;
    for (auto& l : h->audioenc) nets.push_back(&l);
    for (auto& l : h->audiodec) nets.push_back(&l);
    if ((int)nets.size() > DEC_MAXL) { D.why = "persistent decode: too many blocks"; return; }
    DecParams& P = D.tab;
    memset(&P, 0, sizeof(P));
    P.nl = (int)nets.size(); P.n_enc = (int)h->audioenc.size();
    std::vector<int> prow = audiodec_rows(h->audiodec, hp.max_T);
    int nch = 0, off = 0;
    for (int li = 0; li < P.nl; ++li) {
        const LayerDev& l = *nets[li];
        DecLayer& L = P.L[li];
        if (l.kind == K_D || !l.causal || (l.cin % 4) || (l.kind == K_HC && (l.cin != d || l.cout != d)) || l.cout % DEC_NC ||
            (li != 0 && l.cin % 128)) { D.why = "persistent decode: unsupported block " + l.scope; return; }
        L.kind = l.kind == K_HC ? 1 : 0; L.cin = l.cin; L.cout = l.cout; L.ntaps = l.size; L.rate = l.rate; L.act = l.act;
        L.cs = l.cout / DEC_NC; L.ns = L.kind ? 2 * L.cs : (L.cs <= 8 ? 8 : roundup(L.cs, 4));
        if (L.ns != 8 && L.ns != 16 && L.ns != 32) { D.why = "persistent decode: unsupported slice width"; return; }
        L.prow = li >= P.n_enc ? prow[li - P.n_enc] : 1;
        if (L.prow > 1 && (L.cout != 256 || (L.ns != 32 && L.ns != 16) || L.prow > 85)) { D.why = "persistent decode: unsupported receptive field"; return; }
        L.ldin = l.cin;
        const int cinp = roundup(l.cin, 128);                     // AudioEnc C_1: 80 -> 128 zero rows
        if (l.size > 1 && cinp != 256) { D.why = "persistent decode: multi-tap blocks must have 256 input channels"; return; }
        const int K = l.size * cinp;
        L.krows = std::min(K, DEC_SLOT_F / L.ns);                 // k rows per chunk
        const int kr8 = L.krows / 8, sg = 32 / L.ns;
        if (K % L.krows || L.krows % 8 || kr8 * L.ns > DEC_REG_F || kr8 % (8 * sg) || (L.prow > 1 && kr8 % 16)) {
            D.why = "persistent decode: chunk geometry"; return;
        }
        if (L.prow > 1 && (L.prow - 1) + (l.size - 1) * l.rate > DEC_PL_PAD) { D.why = "persistent decode: receptive field too tall"; return; }
        L.ch0 = nch;
        for (int k0 = 0; k0 < K; k0 += L.krows) {
            if (nch >= DEC_MAXCH) { D.why = "persistent decode: too many weight chunks"; return; }
            DecChunk& c = P.C[nch++];
            c.off = off; c.nfl4 = (short)(L.krows * L.ns / 4); c.k0 = (short)k0; c.krows = (short)L.krows; c.layer = (short)li;
            off += L.krows * L.ns;
        }
        L.nch = nch - L.ch0;
        if (li == P.n_enc - 1) P.nch_enc = nch;
        if (L.prow > 1) { if (P.pyr_ch1 == 0) P.pyr_ch0 = L.ch0; P.pyr_ch1 = nch; }
    }
    if (P.L[P.nl - 1].prow != 1 || P.L[P.n_enc].ntaps != 1 || P.nch_enc <= DEC_NSLOT) { D.why = "persistent decode: unexpected AudioDec shape"; return; }
    for (int li = P.n_enc; li < P.nl; ++li)                        // the receptive-field blocks must be a prefix of AudioDec
        if (P.L[li].prow > 1 && li > P.n_enc && P.L[li - 1].prow <= 1) { D.why = "persistent decode: receptive-field blocks not contiguous"; return; }
    P.nch = nch;
    // the receptive-field blocks a second time, as split-fp16 MMA slabs (tensor-core pre-pass): same chunk sizes, appended
    for (int li = 0; li < P.nl; ++li) {
        const DecLayer& L = P.L[li];
        if (L.prow <= 1) continue;
        // kernels_decode.cu instantiates pyr_mma_rows<NS, NTAPS, 1 or 2> for exactly these two shapes -- hc blocks
        // <32, 3, *> and 1x1 convolutions <16, 1, *> -- and stages the first block's input, [ctx | q], from the re-attention
        // (2d channels, lane-strided: d = 256); a new shape needs a new instantiation there, not just a change here
        if (L.krows % 128 || !((L.ns == 32 && L.ntaps == 3) || (L.ns == 16 && L.ntaps == 1)) ||
            (li == P.n_enc && (L.cin != 2 * d || d != 256)) || (li > P.n_enc && L.cin != 256)) {
            D.why = "persistent decode: tensor-core pre-pass geometry"; return;
        }
        for (int c = L.ch0; c < L.ch0 + L.nch; ++c) { P.C[c].off16 = off; off += L.krows * L.ns; }
    }
    P.stream_len = off;
    D.wstream.ensure((size_t)DEC_NC * off * sizeof(float));
    P.wstream = D.wstream.as<float>();
    // LayerNorm parameters [layer][gamma1 | beta1 | gamma2 | beta2][256]; pack_weights copies them in
    D.lnp.ensure((size_t)P.nl * 1024 * sizeof(float));
    CUDA_CHECK(cudaMemset(D.lnp.p, 0, D.lnp.bytes));
    for (int li = 0; li < P.nl; ++li) { P.lnp[li] = D.lnp.as<float>() + (size_t)li * 1024; P.bias[li] = nets[li]->bias; }
    D.tables_ok = true;
    D.max_clusters = decode_max_active_clusters();
    if (D.max_clusters < 1) { D.why = "persistent decode: a 16-CTA cluster with " + std::to_string(decode_smem_bytes()) + " B of shared memory cannot be scheduled"; return; }
    D.ok = true; D.why.clear();
}

// every layer, in the order of the abs-max table: TextEnc, AudioEnc, AudioDec, SSRN
std::vector<LayerDev*> all_layers(H* h) {
    std::vector<LayerDev*> v;
    for (auto* vec : {&h->textenc, &h->audioenc, &h->audiodec, &h->ssrn})
        for (auto& l : *vec) v.push_back(&l);
    return v;
}

void commit_params(H* h) {
    REQUIRE(!h->committed, "parameters already committed on this handle");
    CUDA_CHECK(cudaSetDevice(h->device));
    h->n_params = 0;
    {
        const std::string name = "Text2Mel/TextEnc/embed_1/lookup_table";
        const HostParam& p = need(h, name, {h->hp.vocab_size, h->hp.e});
        h->embed_table = upload(h, p.data);
        h->dev_vec[name] = h->embed_table;
        h->n_params += (int64_t)h->hp.vocab_size * h->hp.e;
    }
    size_t expected = 1;
    for (auto* vec : {&h->textenc, &h->audioenc, &h->audiodec, &h->ssrn})
        for (auto& l : *vec) { commit_layer(h, l); expected += (l.kind == K_HC) ? 6 : 4; }
    if (h->staged.size() != expected) {
        for (auto& kvp : h->staged) {
            const std::string& n = kvp.first;
            bool known = h->dev_vec.count(n) || n.find("/kernel") != std::string::npos;
            if (!known) throw std::runtime_error("unknown variable staged: " + n);
        }
        throw std::runtime_error("staged variable count does not match the path's variable set");
    }
    decode_tables(h);
    h->dec.commit_ok = h->dec.ok; h->dec.commit_why = h->dec.why;
    pack_weights(h, nullptr);
    h->staged.clear();
    h->committed = true;
}

}  // namespace

// The wgmma planes of every block that has them and the persistent decode's weight stream and LayerNorm parameters,
// packed on the device from the layers' fp32 variables as they are now (kernels_pack.cu).  One abs-max reduction over
// every layer, read back, gives the power-of-two scales the host tables hold (LayerDev::TcPack::inv_scale,
// DecParams::inv_scale).  Writes nothing but those planes, that stream and the abs-max slots; synchronises `s`.
void dctts::api::pack_weights(H* h, cudaStream_t s) {
    const std::vector<LayerDev*> layers = all_layers(h);
    const int n = (int)layers.size();
    REQUIRE(n <= PACK_MAXL, "pack_weights: more layers than one abs-max launch takes");
    PackMaxTable t{};
    for (int i = 0; i < n; ++i) { t.W[i] = layers[i]->W; t.n[i] = (long long)layers[i]->size * layers[i]->cin * layers[i]->ldw; }
    t.count = n;
    CUDA_CHECK(cudaMemsetAsync(h->pack_max.p, 0, (size_t)n * sizeof(unsigned), s));
    launch_weight_absmax(t, h->pack_max.as<unsigned>(), s);
    std::vector<float> maxabs((size_t)n);
    CUDA_CHECK(cudaMemcpyAsync(maxabs.data(), h->pack_max.p, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    for (int i = 0; i < n; ++i) {
        LayerDev& l = *layers[i];
        LayerDev::TcPack& p = l.tc;
        if (!p.ok) continue;
        const float scale = weight_scale(maxabs[i]);
        p.inv_scale = 1.f / scale;
        launch_pack_tc(TcPackArgs{l.W, p.Whi, p.Wlo, p.mode, l.cin, l.cout, l.ldw, roundup(l.cin, 64), p.Ktot, p.nrows, p.bn,
                                  p.half, scale}, s);
    }
    auto& D = h->dec;
    if (D.tables_ok) {
        DecParams& P = D.tab;
        const int first = (int)h->textenc.size();                 // AudioEnc's first block in `layers`
        CUDA_CHECK(cudaMemsetAsync(D.wstream.p, 0, (size_t)DEC_NC * P.stream_len * sizeof(float), s));
        for (int li = 0; li < P.nl; ++li) {
            const LayerDev& l = *layers[first + li];
            const DecLayer& L = P.L[li];
            // power-of-two scale of the receptive-field blocks' MMA slabs, as for the block planes
            P.inv_scale[li] = L.prow > 1 ? 1.f / weight_scale(maxabs[first + li]) : 1.f;
            const int cinp = roundup(l.cin, 128);
            launch_pack_decode(DecPackArgs{l.W, D.wstream.as<float>(), P.stream_len, L.kind, l.cin, l.cout, l.ldw, cinp, l.size * cinp,
                                           L.krows, L.ns, L.cs, P.C[L.ch0].off, P.C[L.ch0].off16,
                                           L.prow > 1 ? 1.f / P.inv_scale[li] : 0.f}, s);
            const float* src[4] = {l.g1, l.b1, l.kind == K_HC ? l.g2 : nullptr, l.kind == K_HC ? l.b2 : nullptr};
            for (int q = 0; q < 4; ++q)
                if (src[q]) CUDA_CHECK(cudaMemcpyAsync(D.lnp.as<float>() + (size_t)li * 1024 + q * 256, src[q], (size_t)l.cout * sizeof(float),
                                                        cudaMemcpyDeviceToDevice, s));
        }
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(s));
}

extern "C" {

int dctts_set_param(dctts_handle h, const char* tf_name, const float* data, const int64_t* shape, int32_t rank) {
    return guarded(h, [&] {
        REQUIRE(!h->committed, "parameters already committed");
        REQUIRE(tf_name && data && shape && rank >= 1 && rank <= 4, "dctts_set_param: bad arguments");
        HostParam p;
        size_t n = 1;
        for (int i = 0; i < rank; ++i) { REQUIRE(shape[i] > 0, "dctts_set_param: bad shape"); p.shape.push_back(shape[i]); n *= (size_t)shape[i]; }
        p.data.assign(data, data + n);
        h->staged[tf_name] = std::move(p);
    });
}

int dctts_commit_params(dctts_handle h) {
    return guarded(h, [&] {
        require_no_synth_stream(h, "dctts_commit_params");
        commit_params(h);
        chist_clear(h, "the weights were committed after the last full-sequence chain");
    });
}

int64_t dctts_num_params(dctts_handle h) { return (h && h->committed) ? h->n_params : -1; }

int dctts_refresh_synthesis(dctts_handle h, void* stream) {
    return guarded(h, [&] {
        require_no_synth_stream(h, "dctts_refresh_synthesis");
        REQUIRE(h->committed, "dctts_refresh_synthesis: parameters not committed");
        if (!h->synth_stale) return;
        chist_clear(h, "the weights were repacked after the last full-sequence chain");
        pack_weights(h, S(h, stream));
        CUDA_CHECK(cudaDeviceSynchronize());          // a replay of the captured AR step may still be in flight on another stream
        drop_ar_graph(h);
        h->tensor_path = 1;
        h->dec.ok = h->dec.commit_ok; h->dec.why = h->dec.commit_why;
        h->synth_stale = false;
    });
}

}  // extern "C"
