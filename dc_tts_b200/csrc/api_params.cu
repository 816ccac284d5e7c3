// api_params.cu -- layer tables; parameter staging, split-fp16 packing and the persistent decode's weight stream.
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

// Split-fp16 packing for the wgmma kernel (kernels_tc.cu).  Rows are accumulator columns in
// cluster-slice order (CTA i owns rows [i*bn, (i+1)*bn); for hc / transposed conv its first
// `half` rows are the first LN half, the rest the second), columns are k = tap*cin_pad + ci.
// Weights are multiplied by weight_scale (numerics.cuh); the kernel multiplies the accumulator back.
void pack_tc(H* h, LayerDev& l, const std::vector<float>& W /* [size][cin][ldw] */) {
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
    auto wv = [&](int tap, int ci, int row) -> float {
        const int i = row / p.bn, a = row % p.bn;
        if (p.mode == 0) return row < l.cout ? W[((size_t)tap * l.cin + ci) * l.ldw + row] : 0.f;
        const bool second = a >= p.half;
        const int col = i * p.half + (a % p.half);
        if (p.mode == 1) return W[((size_t)tap * l.cin + ci) * l.ldw + (second ? l.cout + col : col)];
        // transposed conv: k-tap 0 reads x[t] (W0 -> even rows, W1 -> odd rows), k-tap 1 reads x[t-1] (W2 -> even rows)
        if (tap == 0) return W[((size_t)(second ? 1 : 0) * l.cin + ci) * l.ldw + col];
        return second ? 0.f : W[((size_t)2 * l.cin + ci) * l.ldw + col];
    };
    float maxabs = 0.f;
    for (int tap = 0; tap < p.ntaps; ++tap)
        for (int ci = 0; ci < l.cin; ++ci)
            for (int row = 0; row < p.nrows; ++row) maxabs = std::max(maxabs, std::fabs(wv(tap, ci, row)));
    const float scale = weight_scale(maxabs);
    p.inv_scale = 1.f / scale;
    std::vector<__half> hi((size_t)p.nrows * p.Ktot, __float2half_rn(0.f)), lo(hi);
    for (int row = 0; row < p.nrows; ++row)
        for (int tap = 0; tap < p.ntaps; ++tap)
            for (int ci = 0; ci < l.cin; ++ci) {
                const size_t idx = (size_t)row * p.Ktot + (size_t)tap * cin_pad + ci;
                split_f16(wv(tap, ci, row) * scale, hi[idx], lo[idx]);
            }
    p.Whi = upload(h, hi);
    p.Wlo = upload(h, lo);
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
    if (l.scope.compare(0, 14, "Text2Mel/Audio") == 0) l.hostW = W;
    pack_tc(h, l, W);
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
// (+ zero columns up to a multiple of 4).
void pack_decode(H* h) {
    auto& D = h->dec;
    D.ok = false;
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
    // streams: chunk = 8 warp regions, region w = rows [w*kr8, (w+1)*kr8) as [k/4][column][4] (32-column slices: pair-split, below)
    std::vector<float> st((size_t)DEC_NC * off, 0.f);
    for (int li = 0; li < P.nl; ++li) {                              // power-of-two scale per receptive-field block (as pack_tc)
        const LayerDev& l = *nets[li]; const DecLayer& L = P.L[li];
        P.inv_scale[li] = 1.f;
        if (L.prow <= 1) continue;
        float maxabs = 0.f;
        for (size_t i = 0; i < l.hostW.size(); ++i) maxabs = std::max(maxabs, std::fabs(l.hostW[i]));
        P.inv_scale[li] = 1.f / weight_scale(maxabs);
    }
    for (int r = 0; r < DEC_NC; ++r)
        for (int li = 0; li < P.nl; ++li) {
            const LayerDev& l = *nets[li]; const DecLayer& L = P.L[li];
            REQUIRE(!l.hostW.empty(), "persistent decode: host weights missing");
            const int cinp = roundup(l.cin, 128), kr8 = L.krows / 8;
            auto column = [&](int n) -> int {
                if (L.kind) return n < L.cs ? r * L.cs + n : l.cout + r * L.cs + (n - L.cs);
                return n < L.cs ? r * L.cs + n : -1;
            };
            for (int c = L.ch0; c < L.ch0 + L.nch; ++c) {
                const DecChunk& ch = P.C[c];
                float* dst = st.data() + (size_t)r * off + ch.off;
                for (int kc = 0; kc < ch.krows; ++kc) {
                    const int k = ch.k0 + kc, tap = k / cinp, ci = k % cinp;
                    if (ci >= l.cin) continue;
                    const int w = kc / kr8, kk = kc % kr8;
                    const float* wrow = l.hostW.data() + ((size_t)tap * l.cin + ci) * l.ldw;
                    for (int n = 0; n < L.ns; ++n) {
                        const int col = column(n);
                        if (col < 0) continue;
                        // 32-column slices: pair-split layout per 8-k block [column parity][k-group][column pair][4 k]
                        // (gemv_warp32); narrower slices: [k/4][column][4]
                        const size_t idx = L.ns == 32 ? (size_t)(kk / 8) * 256 + ((size_t)((n & 1) * 2 + (kk / 4) % 2) * 16 + (n >> 1)) * 4 + (kk % 4)
                                                      : ((size_t)(kk / 4) * L.ns + n) * 4 + (kk % 4);
                        dst[(size_t)w * kr8 * L.ns + idx] = wrow[col];
                    }
                }
                if (L.prow <= 1) continue;
                // the same rows as MMA slabs of 16 k: [plane hi | lo][k8 group][column][8 halfs], 16*ns floats per slab, in k order
                // (slab s of the chunk sits at float offset s*16*ns: region w of the chunk = slabs [w*spr, (w+1)*spr))
                __half* d16 = reinterpret_cast<__half*>(st.data() + (size_t)r * off + ch.off16);
                const float scale = 1.f / P.inv_scale[li];
                for (int kc = 0; kc < ch.krows; ++kc) {
                    const int k = ch.k0 + kc, tap = k / cinp, ci = k % cinp;
                    const int slab = kc / 16, k16 = kc % 16, grp = k16 / 8, e8 = k16 % 8;
                    const float* wrow = l.hostW.data() + ((size_t)tap * l.cin + ci) * l.ldw;
                    for (int n = 0; n < L.ns; ++n) {
                        const int col = column(n);
                        const float v = (col >= 0 && ci < l.cin) ? wrow[col] * scale : 0.f;
                        const size_t base = (size_t)slab * 32 * L.ns;                  // halfs per slab = 2 planes * 2 groups * ns * 8
                        const size_t idx = ((size_t)grp * L.ns + n) * 8 + e8;
                        split_f16(v, d16[base + idx], d16[base + (size_t)2 * L.ns * 8 + idx]);
                    }
                }
            }
        }
    D.wstream.ensure(st.size() * sizeof(float));
    CUDA_CHECK(cudaMemcpy(D.wstream.p, st.data(), st.size() * sizeof(float), cudaMemcpyHostToDevice));
    // LayerNorm parameters [layer][gamma1 | beta1 | gamma2 | beta2][256]
    D.lnp.ensure((size_t)P.nl * 1024 * sizeof(float));
    CUDA_CHECK(cudaMemset(D.lnp.p, 0, D.lnp.bytes));
    for (int li = 0; li < P.nl; ++li) {
        const LayerDev& l = *nets[li];
        float* base = D.lnp.as<float>() + (size_t)li * 1024;
        const float* src[4] = {l.g1, l.b1, l.kind == K_HC ? l.g2 : nullptr, l.kind == K_HC ? l.b2 : nullptr};
        for (int q = 0; q < 4; ++q)
            if (src[q]) CUDA_CHECK(cudaMemcpy(base + q * 256, src[q], (size_t)l.cout * sizeof(float), cudaMemcpyDeviceToDevice));
        P.lnp[li] = base; P.bias[li] = l.bias;
    }
    P.wstream = D.wstream.as<float>();
    for (auto* lp : nets) { lp->hostW.clear(); lp->hostW.shrink_to_fit(); }
    D.max_clusters = decode_max_active_clusters();
    if (D.max_clusters < 1) { D.why = "persistent decode: a 16-CTA cluster with " + std::to_string(decode_smem_bytes()) + " B of shared memory cannot be scheduled"; return; }
    D.ok = true; D.why.clear();
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
    pack_decode(h);
    h->staged.clear();
    h->committed = true;
}

}  // namespace

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

int dctts_commit_params(dctts_handle h) { return guarded(h, [&] { commit_params(h); }); }

int64_t dctts_num_params(dctts_handle h) { return (h && h->committed) ? h->n_params : -1; }

}  // extern "C"
