// api_train.cu -- the training step (forward, backward, Adam), its evaluation, tensor import / export, the conv-GEMM.
#include "api_internal.cuh"

namespace {

// ---------------------------------------------------------------------------- training
// One optimiser step of the reference's trainers (train.py mode "train"): num = 1 Text2Mel (graph :43-68, losses :83-99),
// num = 2 SSRN on ground-truth mels (:69-72, losses :100-108); Adam + clipping :122-132 -- fixed-size batches (BASELINE
// config 5).  Forward = the fp32 block kernels with every pre-LN tensor kept; backward = kernels_train.cu.  Gradients, Adam
// moments and the pointers of all trained variables live in three arenas with identical offsets (the gradient arena is
// what a data-parallel all-reduce sums).  Activation / gradient rows use a leading dimension rounded to 4 floats (F = 1025).
// Buffers are sized for a capacity -- (hp.max_N, hp.max_T) for Text2Mel, (T_in) for SSRN, or more after
// dctts_train_reserve -- and every step runs at its batch's own (N, T) up to it (train_set_shape), as the reference's
// dynamically padded buckets do (data_load.py:122-129).  The capacity only sizes buffers: no kernel of the step reads it.

// The extents of every block for a step at (N, T): TextEnc runs over N text positions, the other networks over T frames,
// doubled by each transposed convolution.  Rows are packed at this shape from the start of each capacity-sized buffer, so
// the dropout mask -- a hash of the flat element index -- is the one of the tensor at the step's shape.
void train_set_shape(H* h, int N, int T) {
    auto& tr = h->tr;
    for (int net = 0; net < (tr.num == 1 ? 3 : 1); ++net) {
        int L = (tr.num == 1 && net == 0) ? N : T;
        for (int i = tr.first[net]; i <= tr.last[net]; ++i) {
            auto& t = tr.layers[i];
            t.L_in = L;
            if (t.l->kind == K_D) L *= 2;
            t.L = L; t.rows = (long long)tr.B * L;
        }
    }
}

// The shape-dependent workspace for steps up to (N, T): saved activations, attention buffers, gradient ping-pong
// buffers and the tensor-core operand planes, and every block's pointers into them.  Grows only; what the buffers held is
// not kept (each step rewrites what it reads).  The arenas -- variables, gradients, Adam moments, the Adam table -- are
// not touched, so neither the optimiser state nor the gradient arena's address changes.
void train_alloc_ws(H* h, int N, int T) {
    auto& tr = h->tr;
    const dctts_hparams& hp = h->hp;
    const int B = tr.B, d = hp.d, num = tr.num;
    size_t pre_f = 0, out_f = 0, g_f = 0, dy_f = 0, wt_f = 0, tca_f = 0, tcb_f = 0, ord_f = 0;
    train_set_shape(h, N, T);                                    // the capacity: every buffer below is sized for it
    for (auto& t : tr.layers) {
        const LayerDev& l = *t.l;
        {   // the ordered mode's partials: the block backward and the weight gradient on either kernel set, whose split
            // counts grow with the rows, so the capacity bounds every step
            ord_f = std::max(ord_f, block_bwd_ordered_floats(t.rows, l.cout, l.kind == K_HC ? 1 : 0));
            WgradArgs w{};
            w.K = l.cin;
            if (l.kind == K_D) {
                w.rows = (long long)B * t.L_in; w.L = t.L_in; w.N = l.cout; w.ntaps = 1;
                ord_f = std::max(ord_f, conv_wgrad_ordered_floats(w));
            } else {
                w.rows = t.rows; w.L = t.L_in; w.N = l.nconv; w.ntaps = l.size;
                ord_f = std::max({ord_f, conv_wgrad_ordered_floats(w), conv_wgrad_tc_ordered_floats(w, B)});
            }
        }
        t.ld_out = roundup(l.cout, 4);
        pre_f += (size_t)t.rows * l.ldw; out_f += (size_t)t.rows * t.ld_out;
        g_f = std::max(g_f, (size_t)t.rows * std::max(t.ld_out, roundup(l.cin, 4)));
        dy_f = std::max(dy_f, (size_t)t.rows * l.ldw);
        wt_f = std::max(wt_f, (size_t)l.size * l.ldw * roundup(l.cin, 4));
        {   // operand planes of the tensor-core GEMMs: activations / gradients (plain and transposed), packed weights
            const size_t rows_in = (size_t)B * t.L_in, cmax = (size_t)roundup(std::max(l.cin, l.ldw), 8);
            tca_f = std::max(tca_f, std::max(rows_in * cmax, (size_t)l.size * B * roundup(l.cin, 8) * roundup(t.L_in, 8)));
            tcb_f = std::max(tcb_f, std::max((size_t)B * cmax * roundup(t.L_in, 8),
                                             (size_t)l.size * roundup(std::max(l.cin, l.ldw) + 255, 256) * roundup(std::max(l.cin, l.ldw), 32)));
        }
    }
    tr.pre.ensure(pre_f * sizeof(float)); tr.out.ensure(out_f * sizeof(float));
    if (num == 1) {
        tr.emb.ensure((size_t)B * N * hp.e * sizeof(float)); tr.R.ensure((size_t)B * T * 2 * d * sizeof(float));
        tr.align.ensure((size_t)B * N * T * sizeof(float)); tr.dS.ensure((size_t)B * T * N * sizeof(float));
        g_f = std::max(g_f, (size_t)B * std::max(N, T) * (size_t)std::max(2 * d, hp.e));
    }
    for (auto& g : tr.gbuf) g.ensure(g_f * sizeof(float));
    tr.dy.ensure(dy_f * sizeof(float)); tr.wT.ensure(wt_f * sizeof(float));
    tr.tc_a_hi.ensure(tca_f * sizeof(__half)); tr.tc_a_lo.ensure(tca_f * sizeof(__half));
    tr.tc_b_hi.ensure(tcb_f * sizeof(__half)); tr.tc_b_lo.ensure(tcb_f * sizeof(__half));
    tr.tc_slots.ensure(2048 * sizeof(unsigned));
    tr.tc = GemmTcWs{};
    tr.tc.a_hi = tr.tc_a_hi.as<__half>(); tr.tc.a_lo = tr.tc_a_lo.as<__half>(); tr.tc.a_elems = tca_f;
    tr.tc.b_hi = tr.tc_b_hi.as<__half>(); tr.tc.b_lo = tr.tc_b_lo.as<__half>(); tr.tc.b_elems = tcb_f;
    tr.tc.slots = tr.tc_slots.as<unsigned>(); tr.tc.n_slots = 2048;
    float* pre = tr.pre.as<float>(); float* out = tr.out.as<float>();
    for (auto& t : tr.layers) {
        t.pre = pre; pre += (size_t)t.rows * t.l->ldw;
        t.out = out; out += (size_t)t.rows * t.ld_out;
    }
    // inputs: each block reads the previous block's output; the first block of a network reads the embedding (TextEnc), the
    // mels shifted by one frame (AudioEnc, train.py:51; set per step), R (AudioDec) or the ground-truth mels (SSRN, per step)
    for (int net = 0; net < (num == 1 ? 3 : 1); ++net)
        for (int i = tr.first[net] + 1; i <= tr.last[net]; ++i) { tr.layers[i].in = tr.layers[i - 1].out; tr.layers[i].ld_in = tr.layers[i - 1].ld_out; }
    if (num == 1) {
        tr.layers[tr.first[0]].in = tr.emb.as<float>(); tr.layers[tr.first[0]].ld_in = hp.e;
        tr.layers[tr.first[2]].in = tr.R.as<float>(); tr.layers[tr.first[2]].ld_in = 2 * d;
    }
    tr.ord_floats = ord_f;
    if (h->opt.train_deterministic) { tr.ord_part.ensure(ord_f * sizeof(float)); tr.ord_dpart.ensure(ORD_LOSS_PARTS * sizeof(double)); }
    tr.N_cap = N; tr.T_cap = T;
}

// The ordered mode's workspace when the option is on (allocated at the first step that needs it), else nullptr: the default
// kernels.  It outlives the step, like the rest of the shape-dependent workspace.
const OrderedWs* train_ordered(H* h) {
    auto& tr = h->tr;
    if (!h->opt.train_deterministic) return nullptr;
    tr.ord_part.ensure(std::max<size_t>(tr.ord_floats, 1) * sizeof(float));
    tr.ord_dpart.ensure(ORD_LOSS_PARTS * sizeof(double));
    tr.ord.part = tr.ord_part.as<float>(); tr.ord.part_elems = tr.ord_floats;
    tr.ord.dpart = tr.ord_dpart.as<double>(); tr.ord.dpart_elems = ORD_LOSS_PARTS;
    return &tr.ord;
}

// The same for one launch of a test aid (dctts_conv_gemm, dctts_block_bwd, dctts_attn_bwd, dctts_train_loss): `floats`
// partial floats and the loss partials in the call's own buffers
const OrderedWs* call_ordered(H* h, DevBuf& part, DevBuf& dpart, size_t floats, OrderedWs& o) {
    if (!h->opt.train_deterministic) return nullptr;
    part.ensure(std::max<size_t>(floats, 1) * sizeof(float));
    dpart.ensure(ORD_LOSS_PARTS * sizeof(double));
    o.part = part.as<float>(); o.part_elems = floats; o.dpart = dpart.as<double>(); o.dpart_elems = ORD_LOSS_PARTS;
    return &o;
}

void train_init(H* h, int B, float rate, int num, int T_in) {
    REQUIRE(h->committed, "dctts_train_init: parameters must be committed first");
    REQUIRE(B >= 1 && rate >= 0.f && rate < 1.f && (num == 1 || num == 2) && T_in >= 1, "dctts_train_init: bad arguments");
    auto& tr = h->tr;
    if (tr.ready && tr.B == B && tr.num == num && tr.T_in == T_in) { tr.rate = rate; return; }
    CUDA_CHECK(cudaDeviceSynchronize());
    mark_synthesis_stale(h);
    tr.ready = false;
    const dctts_hparams& hp = h->hp;
    tr.layers.clear(); tr.tensors.clear();
    std::vector<std::vector<LayerDev>*> nets;
    if (num == 1) nets = {&h->textenc, &h->audioenc, &h->audiodec}; else nets = {&h->ssrn};
    long long n_grad = 0;
    auto reserve = [&](long long n) { long long o = n_grad; n_grad += (n + 3) / 4 * 4; return o; };
    struct Off { long long W, bias, g1, b1, g2, b2; };
    std::vector<Off> offs;
    const long long table_off = num == 1 ? reserve((long long)hp.vocab_size * hp.e) : 0;
    int li = 0;
    for (size_t net = 0; net < nets.size(); ++net) {
        tr.first[net] = li;
        for (auto& l : *nets[net]) {
            H::TrainLayer t;
            t.l = &l; t.li = li++;
            tr.layers.push_back(t);
        }
        tr.last[net] = li - 1;
    }
    tr.B = B; tr.num = num;
    for (auto& t : tr.layers) {
        const LayerDev& l = *t.l;
        Off o{};
        o.W = reserve((long long)l.size * l.cin * l.ldw); o.bias = reserve(l.ldw);
        o.g1 = reserve(l.cout); o.b1 = reserve(l.cout);
        if (l.kind == K_HC) { o.g2 = reserve(l.cout); o.b2 = reserve(l.cout); }
        offs.push_back(o);
    }
    if (num == 1) {                                              // the (max_N, max_T) table whatever the workspace's capacity
        tr.gts.ensure((size_t)hp.max_N * T_in * sizeof(float)); launch_guided_attention(tr.gts.as<float>(), hp.max_N, T_in, h->stream);
    }
    tr.zeros.ensure(4096 * sizeof(float)); CUDA_CHECK(cudaMemset(tr.zeros.p, 0, 4096 * sizeof(float)));
    tr.sums.ensure(4 * sizeof(double));
    tr.grads.ensure(n_grad * sizeof(float)); tr.mom.ensure(n_grad * sizeof(float)); tr.vel.ensure(n_grad * sizeof(float));
    CUDA_CHECK(cudaMemset(tr.grads.p, 0, n_grad * sizeof(float)));
    CUDA_CHECK(cudaMemset(tr.mom.p, 0, n_grad * sizeof(float))); CUDA_CHECK(cudaMemset(tr.vel.p, 0, n_grad * sizeof(float)));
    tr.n_grad = n_grad;
    float* G = tr.grads.as<float>(); float* M = tr.mom.as<float>(); float* V = tr.vel.as<float>();
    std::vector<AdamEntry> entries;
    // layout: 0 = the TF variable's own layout, 1 = [k][cin][ldw] with ldw > n columns, 2 = transposed conv [tap][cin][ldw] vs TF [1][k][cout][cin]
    auto reg = [&](const std::string& name, float* p, long long off, long long n, int layout = 0, int d0 = 0, int d1 = 0, int d2 = 0, int ld = 0) {
        tr.tensors[name] = H::TrainTensor{p, G + off, M + off, V + off, n, layout, d0, d1, d2, ld};
        entries.push_back(AdamEntry{p, G + off, M + off, V + off, n});
        return G + off;
    };
    if (num == 1) tr.d_table = reg("Text2Mel/TextEnc/embed_1/lookup_table", h->embed_table, table_off, (long long)hp.vocab_size * hp.e);
    for (size_t i = 0; i < tr.layers.size(); ++i) {
        auto& t = tr.layers[i]; LayerDev& l = *t.l; const Off& o = offs[i];
        const long long wn = (long long)l.size * l.cin * l.ldw;
        if (l.kind == K_D) {
            t.dW = reg(l.scope + "/conv2d_transpose/kernel", l.W, o.W, wn, 2, l.size, l.cin, l.cout, l.ldw);
            t.dbias = reg(l.scope + "/conv2d_transpose/bias", l.bias, o.bias, l.ldw, l.ldw != l.cout ? 1 : 0, 1, 1, l.cout, l.ldw);
        } else {
            t.dW = reg(l.scope + "/conv1d/kernel", l.W, o.W, wn, l.ldw != l.nconv ? 1 : 0, l.size, l.cin, l.nconv, l.ldw);
            t.dbias = reg(l.scope + "/conv1d/bias", l.bias, o.bias, l.ldw, l.ldw != l.nconv ? 1 : 0, 1, 1, l.nconv, l.ldw);
        }
        const std::string n1 = l.kind == K_HC ? "/H1" : "/normalize";
        t.dg1 = reg(l.scope + n1 + "/gamma", l.g1, o.g1, l.cout); t.db1 = reg(l.scope + n1 + "/beta", l.b1, o.b1, l.cout);
        if (l.kind == K_HC) { t.dg2 = reg(l.scope + "/H2/gamma", l.g2, o.g2, l.cout); t.db2 = reg(l.scope + "/H2/beta", l.b2, o.b2, l.cout); }
    }
    // the first block of AudioEnc (Text2Mel) or of SSRN reads the step's mels: set per step
    if (num == 1) {
        tr.layers[tr.first[1]].ld_in = hp.n_mels; tr.layers[tr.first[1]].extra_shift = -1; tr.layers[tr.first[1]].need_dgrad = false;
    } else {
        tr.layers[0].ld_in = hp.n_mels; tr.layers[0].need_dgrad = false;
    }
    tr.N_cap = tr.T_cap = 0;
    train_alloc_ws(h, num == 1 ? hp.max_N : 0, T_in);
    tr.entries.ensure(entries.size() * sizeof(AdamEntry));
    CUDA_CHECK(cudaMemcpy(tr.entries.p, entries.data(), entries.size() * sizeof(AdamEntry), cudaMemcpyHostToDevice));
    tr.n_entries = (int)entries.size();
    CUDA_CHECK(cudaStreamSynchronize(h->stream));
    tr.B = B; tr.rate = rate; tr.num = num; tr.T_in = T_in; tr.ready = true;
}

// Grow the workspace of the network being trained to at least N text positions (Text2Mel only) and T mel frames.  Never
// shrinks; a no-op when the workspace already fits.  The arenas stay where they are (train_alloc_ws).
void train_reserve(H* h, int N, int T) {
    auto& tr = h->tr;
    REQUIRE(tr.ready, "dctts_train_reserve: call dctts_train_init or dctts_train_init_ssrn first");
    REQUIRE(N >= 0 && T >= 0, "dctts_train_reserve: bad arguments");
    const int n = tr.num == 1 ? std::max(N, tr.N_cap) : 0, t = std::max(T, tr.T_cap);
    if (n == tr.N_cap && t == tr.T_cap) return;
    CUDA_CHECK(cudaDeviceSynchronize());                         // steps still in flight may read the buffers being replaced
    const int n0 = tr.N_cap, t0 = tr.T_cap;
    try {
        train_alloc_ws(h, n, t);
    } catch (...) {                                              // out of memory: back to the old capacity, or no training state
        cudaGetLastError();
        try { train_alloc_ws(h, n0, t0); } catch (...) { tr.ready = false; cudaGetLastError(); }
        throw;
    }
}

void layer_shifts(const LayerDev& l, int extra, int* shifts) {
    const int tot = (l.size - 1) * l.rate, left = l.causal ? tot : tot / 2;
    for (int j = 0; j < l.size; ++j) shifts[j] = j * l.rate - left + extra;
}

DropArgs drop_args(float rate, int li, uint32_t seed) {
    DropArgs d;
    if (rate > 0.f) {
        d.thresh = (uint32_t)std::min<double>((double)rate * 4294967296.0, 4294967295.0);
        d.scale = 1.0f / (1.0f - rate);
    }
    d.layer = (uint32_t)li; d.seed = seed;
    return d;
}

// forward of blocks [first, last], every pre-LN tensor and block output kept
void train_fwd(H* h, Launch& lc, int first, int last, int B, uint32_t seed) {
    auto& tr = h->tr;
    cudaStream_t s = lc.s;
    for (int i = first; i <= last; ++i) {
        auto& t = tr.layers[i]; const LayerDev& l = *t.l;
        ConvArgs c{};
        c.X = t.in; c.ldx = t.ld_in; c.Y = t.pre; c.ldy = l.ldw; c.bias = l.bias; c.K = l.cin; c.N = l.nconv; c.ldw = l.ldw;
        c.win = RowWin{B, t.L_in, t.L_in, nullptr};
        LnArgs n{};
        n.Y = t.pre; n.ldy = l.ldw; n.g1 = l.g1; n.b1 = l.b1; n.g2 = l.g2; n.b2 = l.b2; n.X = t.in; n.ldx = t.ld_in;
        n.out = t.out; n.ldo = t.ld_out; n.C = l.cout; n.mode = l.kind == K_HC ? 1 : 0; n.act = l.kind == K_D ? 0 : l.act;
        n.win = RowWin{B, t.L, t.L, nullptr};
        if (l.kind == K_D) {                                        // modules.py:232-239, like run_deconv
            const size_t tapsz = (size_t)l.cin * l.ldw;
            c.Lout = 2 * t.L_in; c.ostride = 2;
            c.ntaps = 2; c.taps[0] = ConvTap{l.W + 0 * tapsz, 0}; c.taps[1] = ConvTap{l.W + 2 * tapsz, -1}; c.ooff = 0;
            launch_conv_gemm(c, s, 0, false); lc.count();
            c.ntaps = 1; c.taps[0] = ConvTap{l.W + 1 * tapsz, 0}; c.ooff = 1;
            launch_conv_gemm(c, s, 0, false); lc.count();
        } else {
            c.ntaps = l.size;
            int sh[3]; layer_shifts(l, t.extra_shift, sh);
            for (int j = 0; j < l.size; ++j) { c.taps[j].W = l.W + (size_t)j * l.cin * l.ldw; c.taps[j].shift = sh[j]; }
            c.Lout = t.L; c.ostride = 1; c.ooff = 0;
            t.tc_slots = GemmTcSlots{};
            if ((h->opt.train_tc & 1) && conv_gemm_tc_ok(c, tr.tc)) lc.count(launch_conv_gemm_tc(c, tr.tc, s, &t.tc_slots));
            else { launch_conv_gemm(c, s, 0, false); lc.count(); }
        }
        if (tr.rate > 0.f) n.drop = drop_args(tr.rate, t.li, seed);      // the forward mask is applied by the LayerNorm epilogue
        launch_ln_rows(n, s); lc.count();
    }
}

// backward of blocks [first, last]: g_cur holds the gradient w.r.t. the last block's output; returns the buffer with the
// gradient w.r.t. the first block's input (g_cur and g_other alternate)
float* train_bwd(H* h, Launch& lc, int first, int last, int B, uint32_t seed, float* g_cur, float* g_other) {
    auto& tr = h->tr;
    cudaStream_t s = lc.s;
    float* dy = tr.dy.as<float>(); float* wT = tr.wT.as<float>();
    const OrderedWs* ord = train_ordered(h);
    for (int i = last; i >= first; --i) {
        auto& t = tr.layers[i]; const LayerDev& l = *t.l;
        const int cin_p = roundup(l.cin, 4);
        BlockBwdArgs a{};
        a.pre = t.pre; a.ldy = l.ldw; a.gout = g_cur; a.ldg = t.ld_out; a.X = t.in; a.ldx = t.ld_in;
        a.g1 = l.g1; a.b1 = l.b1; a.g2 = l.g2; a.b2 = l.b2; a.dy = dy; a.gin = g_other;
        a.dg1 = t.dg1; a.db1 = t.db1; a.dg2 = t.dg2; a.db2 = t.db2; a.dbias = t.dbias;
        a.rows = t.rows; a.C = l.cout; a.mode = l.kind == K_HC ? 1 : 0; a.act = l.kind == K_D ? 0 : l.act;
        a.drop = drop_args(tr.rate, t.li, seed);
        lc.count(launch_train_block_bwd(a, s, ord));
        if (t.need_dgrad) {
            if (cin_p != l.cin) CUDA_CHECK(cudaMemsetAsync(wT, 0, (size_t)l.size * l.ldw * cin_p * sizeof(float), s));   // zero pad columns
            launch_transpose_w(l.W, wT, l.size, l.cin, l.ldw, l.ldw, cin_p, s); lc.count();
        }
        ConvArgs c{};
        c.Y = g_other; c.ldy = cin_p; c.bias = tr.zeros.as<float>(); c.K = l.nconv; c.N = l.cin; c.ldw = cin_p;
        c.win = RowWin{B, t.L_in, t.L_in, nullptr}; c.Lout = t.L_in; c.ostride = 1; c.ooff = 0;
        const size_t tsz = (size_t)l.ldw * cin_p;                    // one transposed tap: [ldw rows (conv channels)][cin_p]
        WgradArgs w{};
        w.X = t.in; w.ldx = t.ld_in; w.ldw = l.ldw; w.L = t.L_in; w.K = l.cin;
        if (l.kind == K_D) {
            // rows of dy viewed as (B * L_in, 2 ldw): columns [0, C) belong to output row 2t, [ldw, ldw + C) to row 2t + 1.
            // forward: out[2t] = W0 x[t] + W2 x[t-1], out[2t+1] = W1 x[t]
            const size_t tapsz = (size_t)l.cin * l.ldw;
            w.rows = (long long)B * t.L_in; w.ldy = 2 * l.ldw; w.N = l.cout; w.ntaps = 1;
            w.dy = dy;         w.dW = t.dW + 0 * tapsz; w.shifts[0] = 0;  lc.count(launch_conv_wgrad(w, s, ord));
            w.dy = dy;         w.dW = t.dW + 2 * tapsz; w.shifts[0] = -1; lc.count(launch_conv_wgrad(w, s, ord));
            w.dy = dy + l.ldw; w.dW = t.dW + 1 * tapsz; w.shifts[0] = 0;  lc.count(launch_conv_wgrad(w, s, ord));
            if (!t.need_dgrad) continue;
            // dx[u] = dyE[u] W0^T + dyE[u+1] W2^T + dyO[u] W1^T
            c.K = l.cout;
            c.X = dy; c.ldx = 2 * l.ldw; c.ntaps = 2; c.taps[0] = ConvTap{wT + 0 * tsz, 0}; c.taps[1] = ConvTap{wT + 2 * tsz, 1}; c.accumulate = 0;
            launch_conv_gemm(c, s, 0, false); lc.count();
            c.X = dy + l.ldw; c.ntaps = 1; c.taps[0] = ConvTap{wT + 1 * tsz, 0}; c.accumulate = 1;
            launch_conv_gemm(c, s, 0, false); lc.count();
        } else {
            w.rows = t.rows; w.dy = dy; w.ldy = l.ldw; w.dW = t.dW; w.N = l.nconv; w.ntaps = l.size;
            layer_shifts(l, t.extra_shift, w.shifts);
            GemmTcSlots gs{t.tc_slots.x, nullptr};                   // X's abs-max is known from the forward; dy's is computed once, for both gradients
            if ((h->opt.train_tc & 4) && conv_wgrad_tc_ok(w, B, tr.tc)) lc.count(launch_conv_wgrad_tc(w, B, tr.tc, s, &gs, ord));
            else lc.count(launch_conv_wgrad(w, s, ord));
            if (!t.need_dgrad) continue;
            c.X = dy; c.ldx = l.ldw; c.ntaps = l.size;
            for (int j = 0; j < l.size; ++j) { c.taps[j].W = wT + (size_t)j * tsz; c.taps[j].shift = -w.shifts[j]; }
            c.accumulate = a.mode;
            GemmTcSlots gd{gs.w, t.tc_slots.w};                       // operands: dy and W^T (same magnitudes as W)
            if ((h->opt.train_tc & 2) && conv_gemm_tc_ok(c, tr.tc)) lc.count(launch_conv_gemm_tc(c, tr.tc, s, &gd));
            else { launch_conv_gemm(c, s, 0, false); lc.count(); }
        }
        std::swap(g_cur, g_other);
    }
    return g_cur;
}

void train_read_losses(H* h, float* losses_host, double n_el, double n_att, cudaStream_t s) {
    if (!losses_host) return;
    double sums[4];
    CUDA_CHECK(cudaMemcpyAsync(sums, h->tr.sums.p, sizeof(sums), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    losses_host[1] = (float)(sums[0] / n_el);
    losses_host[2] = (float)(sums[1] / n_el);
    losses_host[3] = n_att > 0 ? (float)(sums[2] / n_att) : 0.f;
    losses_host[0] = losses_host[1] + losses_host[2] + losses_host[3];
}

// One Text2Mel step on L (B, N) and mels (B, T, n_mels), packed at that shape, N and T up to the workspace's capacity
// ((hp.max_N, hp.max_T) unless dctts_train_reserve grew it).  The losses are the reference's at this shape (train.py:83-95):
// means over B T n_mels, and the guided-attention sum over the n_lim x t_lim corner of the (max_N, max_T) table divided by
// B n_lim t_lim, n_lim = min(N, max_N), t_lim = min(T, max_T) (the -1 padding of train.py:91 is cropped to the table).  The
// softmax sees N keys and TextEnc's SAME padding the edge at N.
//
// The forward half, shared by the step and dctts_train_eval: the shape checks (before any launch), the forward with the
// step's dropout mask, the attention on the kernel set train_tc selects, and the mel losses into sums[0..1] (their gradient
// into gbuf[0]).  It writes the workspace, the loss sums and the abs-max slots (which every step clears again first), never
// the variables, the gradient arena or the Adam moments.
void train_forward(H* h, Launch& lc, const int* L, int N, const float* mels, int T, int B, uint32_t seed) {
    auto& tr = h->tr;
    cudaStream_t s = lc.s;
    REQUIRE(tr.ready && tr.num == 1 && tr.B == B, "dctts_train_step: call dctts_train_init with this batch size first");
    const dctts_hparams& hp = h->hp;
    REQUIRE(N >= 1 && N <= tr.N_cap && T >= 1 && T <= tr.T_cap,
            "dctts_train_step: N = " + std::to_string(N) + ", T = " + std::to_string(T) + " outside the handle's capacity (1..max_N = " +
            std::to_string(hp.max_N) + ", 1..max_T = " + std::to_string(hp.max_T) +
            (tr.N_cap != hp.max_N || tr.T_cap != hp.max_T ? ", reserved " + std::to_string(tr.N_cap) + " x " + std::to_string(tr.T_cap) : "") +
            "; dctts_train_reserve grows it)");
    const int d = hp.d;
    train_set_shape(h, N, T);
    CUDA_CHECK(cudaMemsetAsync(tr.sums.p, 0, 4 * sizeof(double), s));
    gemm_tc_begin_step(tr.tc, s); tr.tc.probe = h->opt.train_probe;
    tr.layers[tr.first[1]].in = mels;
    launch_embed(L, h->embed_table, tr.emb.as<float>(), B * N, hp.e, s); lc.count();
    train_fwd(h, lc, tr.first[0], tr.last[0], B, seed);
    train_fwd(h, lc, tr.first[1], tr.last[1], B, seed);
    const float* KV = tr.layers[tr.last[0]].out;               // (B, N, 2d): K | V
    const float* Q = tr.layers[tr.last[1]].out;                // (B, T, d)
    // dense softmax attention (training: no window, networks.py:140-153): the wgmma kernel of the synthesis path when the
    // forward GEMMs are on the tensor cores (it does not touch the weights), else one warp per query row on CUDA cores
    if ((h->opt.train_tc & 1) && d == 256)
        run_attention_tc(lc, Q, d, KV, 2 * d, KV + d, 2 * d, B, T, N, nullptr, tr.R.as<float>(), tr.align.as<float>(), nullptr, Planes{});
    else
        run_attention(lc, Q, d, KV, 2 * d, KV + d, 2 * d, RowWin{B, T, T, nullptr}, N, nullptr, tr.R.as<float>(), tr.align.as<float>(),
                      nullptr, nullptr, nullptr);
    train_fwd(h, lc, tr.first[2], tr.last[2], B, seed);
    const auto& lastl = tr.layers[tr.last[2]];
    lc.count(launch_train_loss(lastl.out, lastl.ld_out, mels, tr.gbuf[0].as<float>(), lastl.ld_out, tr.sums.as<double>(), (long long)B * T,
                               hp.n_mels, s, train_ordered(h)));
}

// The attention backward's arguments: gR (B,T,2d) = the gradient of [ctx ; Q], Q (B,T,d), KV (B,N,2d) = [K | V], align
// (B,N,T), the guided-attention table gts (row stride ld_gts) and its (n_lim, t_lim) corner, dS (B,T,N) scratch, gQ (B,T,d),
// gKV (B,N,2d).  The guided-attention loss is sum |A gts| / (B n_lim t_lim) (train.py:91-95).
AttnBwdArgs attn_bwd_args(const float* gR, const float* Q, const float* KV, const float* align, const float* gts, int ld_gts,
                          float* dS, float* gQ, float* gKV, int B, int T, int N, int d, int n_lim, int t_lim) {
    AttnBwdArgs ab{};
    ab.gR = gR; ab.Q = Q; ab.ldq = d; ab.K = KV; ab.V = KV + d; ab.ldkv = 2 * d; ab.align = align;
    ab.gts = gts; ab.ld_gts = ld_gts; ab.dS = dS; ab.gQ = gQ; ab.gKV = gKV;
    ab.B = B; ab.T = T; ab.N = N; ab.d = d; ab.n_lim = n_lim; ab.t_lim = t_lim;
    ab.att_scale = 1.0f / ((float)B * (float)n_lim * (float)t_lim);
    return ab;
}

void train_forward_backward(H* h, const int* L, int N, const float* mels, int T, int B, uint32_t seed, float* losses_host,
                            cudaStream_t s) {
    auto& tr = h->tr;
    const dctts_hparams& hp = h->hp;
    const int d = hp.d;
    Launch lc{h, s};
    train_forward(h, lc, L, N, mels, T, B, seed);
    CUDA_CHECK(cudaMemsetAsync(tr.grads.p, 0, tr.n_grad * sizeof(float), s));
    const float* KV = tr.layers[tr.last[0]].out;
    const float* Q = tr.layers[tr.last[1]].out;
    float* gR = train_bwd(h, lc, tr.first[2], tr.last[2], B, seed, tr.gbuf[0].as<float>(), tr.gbuf[1].as<float>());
    const int n_lim = std::min(N, hp.max_N), t_lim = std::min(T, hp.max_T);      // the crop of train.py:91 to the table
    const AttnBwdArgs ab = attn_bwd_args(gR, Q, KV, tr.align.as<float>(), tr.gts.as<float>(), hp.max_T, tr.dS.as<float>(),
                                         tr.gbuf[2].as<float>(), tr.gbuf[3].as<float>(), B, T, N, d, n_lim, t_lim);
    lc.count(launch_attn_bwd(ab, tr.sums.as<double>(), s, train_ordered(h)));
    float* free_a = (gR == tr.gbuf[0].as<float>()) ? tr.gbuf[1].as<float>() : tr.gbuf[0].as<float>();
    train_bwd(h, lc, tr.first[1], tr.last[1], B, seed, tr.gbuf[2].as<float>(), free_a);
    float* gEmb = train_bwd(h, lc, tr.first[0], tr.last[0], B, seed, tr.gbuf[3].as<float>(), free_a);
    lc.count(launch_embed_bwd(L, gEmb, tr.d_table, B * N, hp.e, hp.vocab_size, s, train_ordered(h)));
    CUDA_CHECK(cudaGetLastError());
    train_read_losses(h, losses_host, (double)B * T * hp.n_mels, (double)B * n_lim * t_lim, s);
}

// An evaluation of the Text2Mel training graph without an update (what the reference's sess.run(g.alignments) or
// sess.run(g.merged) computes on a batch): train_forward, then the guided-attention sum alone, and copies of
// Y = sigmoid(logits) (B, T, n_mels) and the alignments (B, N, T) into the caller's device buffers when they are given.
void train_eval(H* h, const int* L, int N, const float* mels, int T, int B, uint32_t seed, float* Y_out, float* align_out,
                float* losses_host, cudaStream_t s) {
    auto& tr = h->tr;
    const dctts_hparams& hp = h->hp;
    Launch lc{h, s};
    train_forward(h, lc, L, N, mels, T, B, seed);
    const int n_lim = std::min(N, hp.max_N), t_lim = std::min(T, hp.max_T);
    lc.count(launch_attn_loss(tr.align.as<float>(), tr.gts.as<float>(), hp.max_T, tr.sums.as<double>(), B, N, T, n_lim, t_lim, s,
                              train_ordered(h)));
    if (Y_out) {
        const auto& lastl = tr.layers[tr.last[2]];
        launch_sigmoid_rows(lastl.out, lastl.ld_out, Y_out, (long long)B * T, hp.n_mels, s); lc.count();
    }
    if (align_out) CUDA_CHECK(cudaMemcpyAsync(align_out, tr.align.p, (size_t)B * N * T * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CUDA_CHECK(cudaGetLastError());
    train_read_losses(h, losses_host, (double)B * T * hp.n_mels, (double)B * n_lim * t_lim, s);
}

// SSRN (num = 2): ground-truth mels (B, T, n_mels) in, L1 + binary divergence against the linear magnitudes (B, 4T, F), means
// over B 4T F (train.py:100-108); T up to the capacity given to dctts_train_init_ssrn or grown by dctts_train_reserve.
// The forward half, shared by the step and dctts_train_eval_ssrn (same contract as train_forward).
void train_forward_ssrn(H* h, Launch& lc, const float* mels, const float* mags, int B, int T, uint32_t seed) {
    auto& tr = h->tr;
    cudaStream_t s = lc.s;
    REQUIRE(tr.ready && tr.num == 2 && tr.B == B, "dctts_train_step_ssrn: call dctts_train_init_ssrn with this batch size first");
    REQUIRE(T >= 1 && T <= tr.T_cap, "dctts_train_step_ssrn: T = " + std::to_string(T) + " outside the handle's capacity (1.." +
            std::to_string(tr.T_cap) + ", set by dctts_train_init_ssrn" + (tr.T_cap != tr.T_in ? " and dctts_train_reserve)" : ")"));
    train_set_shape(h, 0, T);
    CUDA_CHECK(cudaMemsetAsync(tr.sums.p, 0, 4 * sizeof(double), s));
    gemm_tc_begin_step(tr.tc, s); tr.tc.probe = h->opt.train_probe;
    tr.layers[0].in = mels;
    const int last = (int)tr.layers.size() - 1;
    train_fwd(h, lc, 0, last, B, seed);
    const auto& ll = tr.layers[last];
    lc.count(launch_train_loss(ll.out, ll.ld_out, mags, tr.gbuf[0].as<float>(), ll.ld_out, tr.sums.as<double>(), ll.rows, ll.l->cout, s,
                               train_ordered(h)));
}

void train_forward_backward_ssrn(H* h, const float* mels, const float* mags, int B, int T, uint32_t seed, float* losses_host,
                                 cudaStream_t s) {
    auto& tr = h->tr;
    Launch lc{h, s};
    train_forward_ssrn(h, lc, mels, mags, B, T, seed);
    CUDA_CHECK(cudaMemsetAsync(tr.grads.p, 0, tr.n_grad * sizeof(float), s));
    const int last = (int)tr.layers.size() - 1;
    train_bwd(h, lc, 0, last, B, seed, tr.gbuf[0].as<float>(), tr.gbuf[1].as<float>());
    CUDA_CHECK(cudaGetLastError());
    const auto& ll = tr.layers[last];
    train_read_losses(h, losses_host, (double)ll.rows * ll.l->cout, 0.0, s);
}

// The SSRN counterpart of train_eval: Z = sigmoid(logits) (B, 4T, F) packed from the last block's padded rows
void train_eval_ssrn(H* h, const float* mels, const float* mags, int B, int T, uint32_t seed, float* Z_out, float* losses_host,
                     cudaStream_t s) {
    auto& tr = h->tr;
    Launch lc{h, s};
    train_forward_ssrn(h, lc, mels, mags, B, T, seed);
    const auto& ll = tr.layers.back();
    if (Z_out) { launch_sigmoid_rows(ll.out, ll.ld_out, Z_out, ll.rows, ll.l->cout, s); lc.count(); }
    CUDA_CHECK(cudaGetLastError());
    train_read_losses(h, losses_host, (double)ll.rows * ll.l->cout, 0.0, s);
}

void train_apply(H* h, long long global_step, float lr, cudaStream_t s) {
    auto& tr = h->tr;
    REQUIRE(tr.ready, "dctts_train_apply: no training state");
    mark_synthesis_stale(h);
    const double beta1 = 0.9, beta2 = 0.999, warm = 4000.0;
    const double step = (double)(global_step + 1);
    const double lr_now = (double)(lr > 0.f ? lr : 0.001f) * std::sqrt(warm) * std::min(step * std::pow(warm, -1.5), 1.0 / std::sqrt(step));   // utils.py:141-145
    const double lr_t = lr_now * std::sqrt(1.0 - std::pow(beta2, step)) / (1.0 - std::pow(beta1, step));
    launch_adam(reinterpret_cast<const AdamEntry*>(tr.entries.p), tr.n_entries, (float)lr_t, (float)beta1, (float)beta2, 1e-8f, s);
    h->launches += 1;
    CUDA_CHECK(cudaGetLastError());
}

// Where element i of a trained variable in its TF layout sits on the device, for TrainTensor layouts 1 and 2 (train_init)
size_t device_index(const H::TrainTensor& t, long long i) {
    if (t.layout == 1) return (size_t)(i / t.d2) * t.ld + i % t.d2;          // [d0][d1][d2] <-> [d0][d1][ld]
    const long long ci = i % t.d1, co = i / t.d1 % t.d2, j = i / ((long long)t.d1 * t.d2);
    return ((size_t)j * t.d1 + ci) * t.ld + co;                              // TF [1][tap][cout][cin] <-> device [tap][cin][ld]
}

}  // namespace

// The one place a handle's synthesis is switched off its packed weights: every entry point that writes a variable calls
// it (dctts_train_init, the optimiser update of dctts_train_step / dctts_train_step_ssrn / dctts_train_apply,
// dctts_train_set_tensor of a variable).  The optimiser updates the fp32 weights only, so until dctts_refresh_synthesis
// packs them again synthesis runs on the fp32 kernel set and the graph-per-frame decode, and dctts_set_tensor_path(1) is
// refused.  Cheap when the handle is stale already; otherwise it synchronises the device once to drop the captured AR step.
void dctts::api::mark_synthesis_stale(H* h) {
    chist_clear(h, "training took over the weights after the last full-sequence chain");
    if (h->synth_stale) return;
    if (h->ar_exec) { CUDA_CHECK(cudaDeviceSynchronize()); drop_ar_graph(h); }
    h->tensor_path = 0;
    h->dec.ok = false; h->dec.why = "this handle has been trained: the packed decode stream is stale";
    h->synth_stale = true;
}

extern "C" {

int dctts_conv_gemm(dctts_handle h, int32_t impl, int32_t mode, const float* X, int32_t ldx, int32_t B, int32_t L, int32_t K,
                    const float* Wd, int32_t ldwd, int32_t N, int32_t ntaps, const int32_t* shifts_host, const float* bias,
                    int32_t accumulate, float* out, int32_t ldo, void* stream) {
    DevBuf bufs[5];                                 // the call's own wgmma workspace, freed on every exit
    DevBuf ord_part, ord_dpart;                     // and its ordered-mode partials (option train_deterministic)
    return guarded(h, [&] {
        REQUIRE(impl == 0 || impl == 1, "dctts_conv_gemm: impl must be 0 (fp32 CUDA cores) or 1 (wgmma)");
        REQUIRE(mode == 0 || mode == 1, "dctts_conv_gemm: mode must be 0 (conv) or 1 (weight gradient)");
        REQUIRE(X && Wd && out && shifts_host && B >= 1 && L >= 1 && K >= 1 && N >= 1 && ntaps >= 1 && ntaps <= 3,
                "dctts_conv_gemm: bad arguments");
        REQUIRE(ldx % 4 == 0 && ldwd % 4 == 0 && ldo % 4 == 0, "dctts_conv_gemm: ldx, ldwd and ldo must be multiples of 4");
        REQUIRE(ldx >= K && ldwd >= N && ldo >= N, "dctts_conv_gemm: a pitch is narrower than its tensor's width");
        auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
        REQUIRE(aligned(X) && aligned(Wd) && aligned(out) && aligned(bias), "dctts_conv_gemm: every tensor must be 16-byte aligned");
        if (mode == 0) {
            // the fp32 kernel reads W and bias and writes out over the whole pitch ldwd (ConvArgs: ldy == ldw)
            REQUIRE(bias && ldo == ldwd && (accumulate == 0 || accumulate == 1),
                    "dctts_conv_gemm: mode 0 needs a bias of ldwd floats, ldo == ldwd and accumulate 0 or 1");
        } else {
            REQUIRE(!bias && accumulate == 1, "dctts_conv_gemm: mode 1 adds into out (accumulate = 1) and takes no bias");
        }
        cudaStream_t s = S(h, stream);
        GemmTcWs ws;
        if (impl == 1) {
            const size_t a_el = mode == 0 ? (size_t)B * L * roundup(K, 8) : (size_t)ntaps * B * K * roundup(L, 8);
            const size_t b_el = mode == 0 ? (size_t)roundup(N, 256) * ntaps * roundup(K, 32) : (size_t)B * N * roundup(L, 8);
            for (int i = 0; i < 2; ++i) bufs[i].ensure(a_el * sizeof(__half));
            for (int i = 2; i < 4; ++i) bufs[i].ensure(b_el * sizeof(__half));
            bufs[4].ensure(4 * sizeof(unsigned));
            ws.a_hi = bufs[0].as<__half>(); ws.a_lo = bufs[1].as<__half>(); ws.a_elems = a_el;
            ws.b_hi = bufs[2].as<__half>(); ws.b_lo = bufs[3].as<__half>(); ws.b_elems = b_el;
            ws.slots = bufs[4].as<unsigned>(); ws.n_slots = 4;
            gemm_tc_begin_step(ws, s);
        }
        int launches = 1;
        if (mode == 0) {
            ConvArgs c{};
            c.X = X; c.ldx = ldx; c.Y = out; c.ldy = ldo; c.bias = bias; c.K = K; c.N = N; c.ldw = ldwd;
            c.ntaps = ntaps;
            for (int j = 0; j < ntaps; ++j) c.taps[j] = ConvTap{Wd + (size_t)j * K * ldwd, shifts_host[j]};
            c.win = RowWin{B, L, L, nullptr}; c.Lout = L; c.ostride = 1; c.ooff = 0; c.accumulate = accumulate;
            if (impl == 0) launch_conv_gemm(c, s, 0, false);
            else {
                REQUIRE(conv_gemm_tc_ok(c, ws), "dctts_conv_gemm: conv_gemm_tc_ok does not hold for this call");
                launches = launch_conv_gemm_tc(c, ws, s);
            }
        } else {
            WgradArgs w{};
            w.X = X; w.ldx = ldx; w.dy = Wd; w.ldy = ldwd; w.dW = out; w.ldw = ldo;
            w.rows = (long long)B * L; w.L = L; w.K = K; w.N = N; w.ntaps = ntaps;
            for (int j = 0; j < ntaps; ++j) w.shifts[j] = shifts_host[j];
            OrderedWs o;
            const OrderedWs* ord = call_ordered(h, ord_part, ord_dpart, impl == 0 ? conv_wgrad_ordered_floats(w) : conv_wgrad_tc_ordered_floats(w, B), o);
            if (impl == 0) launches = launch_conv_wgrad(w, s, ord);
            else {
                REQUIRE(conv_wgrad_tc_ok(w, B, ws), "dctts_conv_gemm: conv_wgrad_tc_ok does not hold for this call");
                launches = launch_conv_wgrad_tc(w, B, ws, s, nullptr, ord);
            }
        }
        h->launches += launches;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(s));      // before the workspace is freed
    });
}

int dctts_block_fwd(dctts_handle h, int32_t mode, int32_t act, int64_t rows, int32_t C, const float* pre, int32_t ldy,
                    const float* X, int32_t ldx, const float* ln, float dropout_rate, int32_t layer, uint32_t seed, float* out,
                    int32_t ldo, void* stream) {
    return guarded(h, [&] {
        REQUIRE(mode == 0 || mode == 1, "dctts_block_fwd: mode must be 0 (conv1d / transposed conv) or 1 (highway)");
        REQUIRE(act == 0 || act == 1, "dctts_block_fwd: act must be 0 (none) or 1 (ReLU)");
        REQUIRE(rows >= 1 && rows < (1ll << 31) && C >= 1 && layer >= 0 && dropout_rate >= 0.f && dropout_rate < 1.f,
                "dctts_block_fwd: bad arguments");
        REQUIRE(pre && ln && out && (mode == 0 || X), "dctts_block_fwd: pre, ln, out (and X for a highway block) are required");
        REQUIRE(ldy >= (mode == 1 ? 2 * C : C) && ldo >= C && (mode == 0 || ldx >= C),
                "dctts_block_fwd: a pitch is narrower than its tensor's width");
        // the LayerNorm epilogue of train_fwd: one launch_ln_rows over the rows, the step's dropout mask from drop_args
        LnArgs n{};
        n.Y = pre; n.ldy = ldy; n.g1 = ln; n.b1 = ln + C; n.g2 = ln + 2 * C; n.b2 = ln + 3 * C; n.X = X; n.ldx = ldx;
        n.out = out; n.ldo = ldo; n.C = C; n.mode = mode; n.act = act; n.win = RowWin{1, (int)rows, (int)rows, nullptr};
        if (dropout_rate > 0.f) n.drop = drop_args(dropout_rate, layer, seed);
        cudaStream_t s = S(h, stream);
        launch_ln_rows(n, s); h->launches++;           // refuses a width past the widest LayerNorm kernel before launching
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_block_bwd(dctts_handle h, int32_t mode, int32_t act, int64_t rows, int32_t C, const float* pre, int32_t ldy,
                    const float* gout, int32_t ldg, const float* X, int32_t ldx, const float* ln, float dropout_rate, int32_t layer,
                    uint32_t seed, float* dy, float* gin, float* dparams, void* stream) {
    DevBuf ord_part, ord_dpart;                     // the call's ordered-mode partials (option train_deterministic)
    return guarded(h, [&] {
        REQUIRE(mode == 0 || mode == 1, "dctts_block_bwd: mode must be 0 (conv1d / transposed conv) or 1 (highway)");
        REQUIRE(act == 0 || act == 1, "dctts_block_bwd: act must be 0 (none) or 1 (ReLU)");
        REQUIRE(rows >= 1 && C >= 1 && layer >= 0 && dropout_rate >= 0.f && dropout_rate < 1.f, "dctts_block_bwd: bad arguments");
        const int nconv = mode == 1 ? 2 * C : C;
        REQUIRE(pre && gout && ln && dy && dparams && (mode == 0 || (X && gin)),
                "dctts_block_bwd: pre, gout, ln, dy, dparams (and X, gin for a highway block) are required");
        REQUIRE(ldy >= nconv && ldg >= C && (mode == 0 || ldx >= C), "dctts_block_bwd: a pitch is narrower than its tensor's width");
        cudaStream_t s = S(h, stream);
        BlockBwdArgs a{};
        a.pre = pre; a.ldy = ldy; a.gout = gout; a.ldg = ldg; a.X = X; a.ldx = ldx;
        a.g1 = ln; a.b1 = ln + C; a.g2 = ln + 2 * C; a.b2 = ln + 3 * C; a.dy = dy; a.gin = gin;
        a.dg1 = dparams; a.db1 = dparams + C; a.dg2 = dparams + 2 * C; a.db2 = dparams + 3 * C; a.dbias = dparams + 4 * C;
        a.rows = rows; a.C = C; a.mode = mode; a.act = act;
        a.drop = drop_args(dropout_rate, layer, seed);
        OrderedWs o;
        const OrderedWs* ord = call_ordered(h, ord_part, ord_dpart, block_bwd_ordered_floats(rows, C, mode), o);
        h->launches += launch_train_block_bwd(a, s, ord);   // refuses a width no kernel instantiation covers before launching
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_attn_bwd(dctts_handle h, const float* gR, const float* Q, const float* KV, const float* align, const float* gts,
                   int32_t ld_gts, int32_t B, int32_t T, int32_t N, int32_t n_lim, int32_t t_lim, float* gQ, float* gKV, double* sums,
                   void* stream) {
    DevBuf dS;                                      // the call's own dS scratch, freed on every exit
    DevBuf ord_part, ord_dpart;                     // and its ordered-mode partials (option train_deterministic)
    return guarded(h, [&] {
        REQUIRE(gR && Q && KV && align && gts && gQ && gKV && sums && B >= 1 && T >= 1 && N >= 1, "dctts_attn_bwd: bad arguments");
        AttnBwdArgs a = attn_bwd_args(gR, Q, KV, align, gts, ld_gts, nullptr, gQ, gKV, B, T, N, h->hp.d, n_lim, t_lim);
        check_attn_bwd(a);                         // d and the crop, before the scratch is allocated
        dS.ensure((size_t)B * T * N * sizeof(float));
        a.dS = dS.as<float>();
        cudaStream_t s = S(h, stream);
        OrderedWs o;
        h->launches += launch_attn_bwd(a, sums, s, call_ordered(h, ord_part, ord_dpart, 0, o));
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(s));      // before the scratch is freed
    });
}

int dctts_train_loss(dctts_handle h, const float* logits, int32_t ldl, const float* target, int64_t rows, int32_t C, float* dlogits,
                     int32_t ldg, float* Y, double* sums, void* stream) {
    DevBuf ord_part, ord_dpart;                     // the call's ordered-mode partials (option train_deterministic)
    return guarded(h, [&] {
        REQUIRE(logits && target && dlogits && sums && rows >= 1 && C >= 1, "dctts_train_loss: bad arguments");
        REQUIRE(ldl >= C && ldg >= C, "dctts_train_loss: a pitch is narrower than its tensor's width");
        cudaStream_t s = S(h, stream);
        OrderedWs o;
        h->launches += launch_train_loss(logits, ldl, target, dlogits, ldg, sums, rows, C, s, call_ordered(h, ord_part, ord_dpart, 0, o));
        if (Y) { launch_sigmoid_rows(logits, ldl, Y, rows, C, s); h->launches += 1; }
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int dctts_train_init(dctts_handle h, int32_t B, float dropout_rate) {
    return guarded(h, [&] { require_no_synth_stream(h, "dctts_train_init"); train_init(h, B, dropout_rate, 1, h->hp.max_T); });
}

int dctts_train_step_shaped(dctts_handle h, const int32_t* L, int32_t N, const float* mels, int32_t T, int32_t B, int64_t global_step,
                            uint32_t seed, float lr, int32_t apply, float* losses_host, void* stream) {
    return guarded(h, [&] {
        require_no_synth_stream(h, "dctts_train_step_shaped");
        REQUIRE(L && mels && B >= 1 && global_step >= 0, "dctts_train_step: bad arguments");
        cudaStream_t s = S(h, stream);
        train_forward_backward(h, reinterpret_cast<const int*>(L), N, mels, T, B, seed, losses_host, s);
        if (apply) train_apply(h, global_step, lr, s);
    });
}

int dctts_train_step(dctts_handle h, const int32_t* L, const float* mels, int32_t B, int64_t global_step, uint32_t seed, float lr,
                     int32_t apply, float* losses_host, void* stream) {
    return dctts_train_step_shaped(h, L, h ? h->hp.max_N : 0, mels, h ? h->hp.max_T : 0, B, global_step, seed, lr, apply, losses_host, stream);
}

int dctts_train_eval(dctts_handle h, const int32_t* L, int32_t N, const float* mels, int32_t T, int32_t B, uint32_t seed,
                     float* Y_out, float* align_out, float* losses_host, void* stream) {
    return guarded(h, [&] {
        REQUIRE(L && mels && B >= 1, "dctts_train_eval: bad arguments");
        train_eval(h, reinterpret_cast<const int*>(L), N, mels, T, B, seed, Y_out, align_out, losses_host, S(h, stream));
    });
}

int dctts_train_eval_ssrn(dctts_handle h, const float* mels, const float* mags, int32_t B, int32_t T, uint32_t seed, float* Z_out,
                          float* losses_host, void* stream) {
    return guarded(h, [&] {
        REQUIRE(mels && mags && B >= 1, "dctts_train_eval_ssrn: bad arguments");
        train_eval_ssrn(h, mels, mags, B, T, seed, Z_out, losses_host, S(h, stream));
    });
}

int dctts_train_apply(dctts_handle h, int64_t global_step, float lr, void* stream) {
    return guarded(h, [&] { require_no_synth_stream(h, "dctts_train_apply"); REQUIRE(global_step >= 0, "dctts_train_apply: bad step"); train_apply(h, global_step, lr, S(h, stream)); });
}

int dctts_train_reserve(dctts_handle h, int32_t N, int32_t T) {
    return guarded(h, [&] { require_no_synth_stream(h, "dctts_train_reserve"); train_reserve(h, N, T); });
}

int dctts_train_capacity(dctts_handle h, int32_t* N, int32_t* T) {
    return guarded(h, [&] {
        REQUIRE(h->tr.ready && N && T, "dctts_train_capacity: no training state");
        *N = h->tr.num == 1 ? h->tr.N_cap : 0; *T = h->tr.T_cap;
    });
}

int dctts_train_grads(dctts_handle h, float** grads, int64_t* count) {
    return guarded(h, [&] {
        REQUIRE(h->tr.ready && grads && count, "dctts_train_grads: no training state");
        *grads = h->tr.grads.as<float>(); *count = h->tr.n_grad;
    });
}

int dctts_train_init_ssrn(dctts_handle h, int32_t B, int32_t T, float dropout_rate) {
    return guarded(h, [&] { require_no_synth_stream(h, "dctts_train_init_ssrn"); train_init(h, B, dropout_rate, 2, T); });
}

int dctts_train_step_ssrn_shaped(dctts_handle h, const float* mels, const float* mags, int32_t B, int32_t T, int64_t global_step,
                                 uint32_t seed, float lr, int32_t apply, float* losses_host, void* stream) {
    return guarded(h, [&] {
        require_no_synth_stream(h, "dctts_train_step_ssrn_shaped");
        REQUIRE(mels && mags && B >= 1 && global_step >= 0, "dctts_train_step_ssrn: bad arguments");
        cudaStream_t s = S(h, stream);
        train_forward_backward_ssrn(h, mels, mags, B, T, seed, losses_host, s);
        if (apply) train_apply(h, global_step, lr, s);
    });
}

int dctts_train_step_ssrn(dctts_handle h, const float* mels, const float* mags, int32_t B, int64_t global_step, uint32_t seed, float lr,
                          int32_t apply, float* losses_host, void* stream) {
    const int32_t T = h ? h->tr.T_in : 0;              // the capacity given to dctts_train_init_ssrn
    return dctts_train_step_ssrn_shaped(h, mels, mags, B, T, global_step, seed, lr, apply, losses_host, stream);
}

int dctts_train_tensor(dctts_handle h, const char* tf_name, int32_t what, float* host_out, int64_t count) {
    return guarded(h, [&] {
        REQUIRE(h->tr.ready && tf_name && host_out && what >= 0 && what <= 3, "dctts_train_tensor: bad arguments");
        auto it = h->tr.tensors.find(tf_name);
        REQUIRE(it != h->tr.tensors.end(), "dctts_train_tensor: not a variable of the network being trained");
        const auto& t = it->second;
        const long long logical = t.layout == 0 ? t.n : (long long)t.d0 * t.d1 * t.d2;
        REQUIRE(count == logical, "dctts_train_tensor: element count mismatch");
        const float* src = what == 0 ? t.p : what == 1 ? t.g : what == 2 ? t.m : t.v;
        CUDA_CHECK(cudaDeviceSynchronize());
        if (t.layout == 0) {
            CUDA_CHECK(cudaMemcpy(host_out, src, (size_t)count * sizeof(float), cudaMemcpyDeviceToHost));
            return;
        }
        std::vector<float> tmp((size_t)t.n);
        CUDA_CHECK(cudaMemcpy(tmp.data(), src, tmp.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (long long i = 0; i < count; ++i) host_out[i] = tmp[device_index(t, i)];
    });
}

// Inverse of dctts_train_tensor: upload a variable (what = 0), its Adam first (2) or second (3) moment from the TF layout --
// what Supervisor's restore does for a resumed run (train.py:144; ADVICE r1: training could not resume).
int dctts_train_set_tensor(dctts_handle h, const char* tf_name, int32_t what, const float* host_in, int64_t count) {
    return guarded(h, [&] {
        require_no_synth_stream(h, "dctts_train_set_tensor");
        REQUIRE(h->tr.ready && tf_name && host_in && (what == 0 || what == 2 || what == 3), "dctts_train_set_tensor: bad arguments");
        auto it = h->tr.tensors.find(tf_name);
        REQUIRE(it != h->tr.tensors.end(), "dctts_train_set_tensor: not a variable of the network being trained");
        const auto& t = it->second;
        const long long logical = t.layout == 0 ? t.n : (long long)t.d0 * t.d1 * t.d2;
        REQUIRE(count == logical, "dctts_train_set_tensor: element count mismatch");
        float* dst = what == 0 ? t.p : what == 2 ? t.m : t.v;
        CUDA_CHECK(cudaDeviceSynchronize());
        if (what == 0) mark_synthesis_stale(h);
        if (t.layout == 0) {
            CUDA_CHECK(cudaMemcpy(dst, host_in, (size_t)count * sizeof(float), cudaMemcpyHostToDevice));
            return;
        }
        std::vector<float> tmp((size_t)t.n, 0.f);
        for (long long i = 0; i < count; ++i) tmp[device_index(t, i)] = host_in[i];
        CUDA_CHECK(cudaMemcpy(dst, tmp.data(), tmp.size() * sizeof(float), cudaMemcpyHostToDevice));
    });
}

}  // extern "C"
