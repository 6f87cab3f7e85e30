// MADNet engine: forward, MAD / FULL backward and momentum update (see engine.h).
//
// Graph restated from the reference (never copied): pyramid encoder Nets/MadNet.py:173-249, per-level
// warp -> correlation -> 6-conv estimator loop :251-351, context network :122-171, outputs :68-71,:362-364;
// train-op structure Stereo_Online_Adaptation.py:87-128 (MAD: one module per step with gradients cut between
// levels by `bulkhead`; FULL: everything, gradients also flow through the up-sampled disparities).
#include <nvtx3/nvToolsExt.h>

#include "engine.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace ms {

static const int PYR_CH[13] = {3, 16, 16, 32, 32, 64, 64, 96, 96, 128, 128, 192, 192};
static const int EST_CH[6] = {128, 128, 96, 64, 32, 1};
static const int CTX_CH[7] = {128, 128, 128, 96, 64, 32, 1};
static const int CTX_RATE[7] = {1, 2, 4, 8, 16, 1, 1};
static const float MAD_ALPHA = 0.2f;

static inline int pad4(int c) { return (c + 3) / 4 * 4; }
static inline int feat_of(int k) { return 2 * k; }
static inline int est_layer(int k, int j) { return 12 + (6 - k) * 6 + (j - 1); }
static inline int ctx_layer(int j) { return 42 + (j - 1); }

static void same_pad(int in, int k, int s, int d, int& out, int& before) {
    int keff = (k - 1) * d + 1;
    out = (in + s - 1) / s;
    int total = std::max((out - 1) * s + keff - in, 0);
    before = total / 2;
}

Engine::Engine()
    : net(0), B(1), H(0), W(0), Hp(0), Wp(0), radius_d(2), corr_stride(1), warping(1), n_groups(0), n_params(0),
      Wt(nullptr), Gr(nullptr), Mo(nullptr), ws(nullptr), ws_floats(0), bound(false), wT(nullptr), wT_floats(0),
      wg_ws(nullptr), wg_ws_floats(0), rs_tmp(nullptr), rs_tmp_floats(0), loss_ws(nullptr), loss_ws_floats(0),
      scalars(nullptr), gt(nullptr), proxy(nullptr), loss_kind(0), proxy_w_full(0.01f), proxy_w_module(0.1f), profiling(0), prof_capturing(false), prof_event_overhead_ms(0.f) {
    prof_reset();
    splitk[0] = splitk[1] = SplitK{nullptr, nullptr, nullptr}; on_branch = 0; weights_dirty = true;
    gstream = nullptr; ev_in = nullptr; ev_out = nullptr;
    wstream = nullptr; ev_fork = nullptr; ev_join = nullptr; wstream_dirty = false;
    bstream = nullptr; ev_bfork = nullptr; ev_bjoin = nullptr; loss_full_ws = nullptr;
    wg_xp.hi = wg_xp.lo = nullptr; wg_xp.cs = 0; wg_xp.fmt = 0; wg_xp.scale = 1.f; wg_xp_halfs = 0;
    act_scale = 0.f;
    bf_jobs_dev = nullptr; bf_max_total = 0;
    dp_rank = 0; dp_world = 1; dp_connected = false; dp_xbuf = nullptr; dp_state = nullptr; dp_cap_floats = 0;
    opt_kind = 0; adam_b1 = adam_b2 = adam_eps = 0.f; adam_v = nullptr; adam_powers = nullptr;
    rect_map_l = rect_map_r = nullptr; rect_h = rect_w = 0; rect_scratch = nullptr;
    rs_scale = 1; rs_fresh = false; memset(rs_tab, 0, sizeof rs_tab);
}

void Engine::drop_graphs() {
    for (auto& g : graphs) cudaGraphExecDestroy(g.second.exec);
    graphs.clear();
}

int Engine::set_optimizer(int kind, float beta1, float beta2, float eps, float* v, float* powers) {
    MS_REQUIRE(kind == 0 || kind == 1, "set_optimizer: kind must be 0 (momentum) or 1 (adam)");
    if (kind == 1) {
        MS_REQUIRE(v && powers, "set_optimizer: Adam needs the second-moment arena and the two beta powers");
        MS_REQUIRE((reinterpret_cast<uintptr_t>(v) & 15) == 0, "set_optimizer: the second-moment arena must be 16B aligned");
        MS_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f, "set_optimizer: bad Adam constants");
    } else {
        beta1 = beta2 = eps = 0.f; v = nullptr; powers = nullptr;
    }
    if (kind != opt_kind || beta1 != adam_b1 || beta2 != adam_b2 || eps != adam_eps || v != adam_v || powers != adam_powers)
        drop_graphs();          // the update kernels are baked into the step graphs
    opt_kind = kind; adam_b1 = beta1; adam_b2 = beta2; adam_eps = eps; adam_v = v; adam_powers = powers;
    return 0;
}

int Engine::ensure_planes(const TView& v, const ActPlanes* pl, cudaStream_t st) {
    if (fresh.count(v.p)) return 0;
    MS_REQUIRE(pl != nullptr, "ensure_planes: tensor has no 16-bit planes");
    if (split_planes(v, *pl, st)) return -1;
    fresh.insert(v.p);
    return 0;
}
// after a kernel wrote v: its planes are fresh if and only if the kernel wrote them too
void Engine::planes_written(const TView& v, const ActPlanes* pl, bool written) {
    if (written && pl) fresh.insert(v.p);
    else fresh.erase(v.p);
}

// SAME padding of the layer's convolution from `in` to `out` (a transposed layer: of the stride-s conv that maps its
// output back to its input); false if `out` is not the size that convolution produces
static bool conv_pads(const ConvLayer& L, const TView& in, const TView& out, int& pt, int& pl) {
    int oh, ow;
    same_pad(in.h, L.kh, L.stride, L.dil, oh, pt);
    same_pad(in.w, L.kw, L.stride, L.dil, ow, pl);
    return oh == out.h && ow == out.w;
}

bool conv_fwd_geom(const ConvLayer& L, const TView& x, const TView& y, ConvGemm& p) {
    p = ConvGemm{};
    p.x = x; p.y = y; p.kh = L.kh; p.kw = L.kw;
    p.alpha = L.alpha; p.mask_alpha = 1.f;
    int pt, pl;
    const bool ok = L.transposed ? conv_pads(L, y, x, pt, pl) : conv_pads(L, x, y, pt, pl);
    if (!L.transposed) { p.mul = L.stride; p.off_y = -pt; p.off_x = -pl; p.step = L.dil; p.div = 1; }
    else { p.mul = 1; p.off_y = pt; p.off_x = pl; p.step = -1; p.div = L.stride; }
    return ok && x.c == L.cin && y.c == L.cout;
}
// input gradient: the gather of dpre (a transposed layer: the stride-s conv of dpre with its canonical weights)
bool conv_dgrad_geom(const ConvLayer& L, const TView& dpre, const TView& dx, ConvGemm& p) {
    p = ConvGemm{};
    p.x = dpre; p.y = dx; p.kh = L.kh; p.kw = L.kw;
    p.alpha = 1.f; p.mask_alpha = 1.f;
    int pt, pl;
    const bool ok = L.transposed ? conv_pads(L, dpre, dx, pt, pl) : conv_pads(L, dx, dpre, pt, pl);
    if (L.transposed) { p.mul = L.stride; p.off_y = -pt; p.off_x = -pl; p.step = 1; p.div = 1; }
    else { p.mul = 1; p.off_y = pt; p.off_x = pl; p.step = -L.dil; p.div = L.stride; }
    return ok && dpre.c == L.cout && dx.c == L.cin;
}
// weight gradient (a transposed layer: of the stride-s conv from its output-sized dpre to its input x)
bool conv_wgrad_geom(const ConvLayer& L, const TView& x, const TView& dpre, ConvWgrad& q) {
    q = ConvWgrad{};
    q.x = L.transposed ? dpre : x; q.dy = L.transposed ? x : dpre;
    q.kh = L.kh; q.kw = L.kw; q.stride = L.stride; q.dil = L.dil;
    return conv_pads(L, q.x, q.dy, q.pad_t, q.pad_l) && x.c == L.cin && dpre.c == L.cout;
}

// The engine's pointers on top of that geometry, shared by the planner and the dispatch so that both put the same
// question to the kernels' predicates.
bool Engine::fwd_args(int li, ConvGemm& p) const {
    const ConvLayer& L = layers[li];
    const bool ok = conv_fwd_geom(L, plan[li].x, plan[li].y, p);
    // canonical W of a transposed layer is [tap][cout][cin]; the gather GEMM wants [tap][K=cin][N=cout] (transpose_taps)
    p.wmat = L.transposed ? wT : Wt + L.w_off; p.bias = Wt + L.b_off;
    p.part = sk().gemm_part; p.part_floats = conv_gemm_part_floats();
    return ok;
}
bool Engine::dgrad_args(int li, ConvGemm& p) const {
    const ConvLayer& L = layers[li];
    const bool ok = conv_dgrad_geom(L, plan[li].dpre, plan[li].dx, p);
    p.wmat = Wt + L.w_off;
    p.part = sk().gemm_part; p.part_floats = conv_gemm_part_floats();
    return ok;
}
bool Engine::wgrad_args(int li, ConvWgrad& q) const {
    const ConvLayer& L = layers[li];
    const bool ok = conv_wgrad_geom(L, plan[li].x, plan[li].dpre, q);
    q.dw = Gr + L.w_off; q.db = L.transposed ? nullptr : Gr + L.b_off;      // a transposed layer's bias: bias_grad
    q.workspace = wg_ws; q.workspace_floats = wg_ws_floats;
    return ok;
}

void Engine::prof_reset() {
    for (int i = 0; i < N_CAT; ++i) { cat_ms[i] = 0; cat_macs[i] = 0; cat_bytes[i] = 0; cat_calls[i] = 0; }
    for (int d = 0; d < 3; ++d) { layer_ms[d].assign(layers.size(), 0.0); layer_calls[d].assign(layers.size(), 0); }
}
void Engine::prof_begin(int cat, cudaStream_t st, int layer) {
    if (!profiling || (profiling == 2 && !prof_capturing)) return;
    Span s; s.cat = cat; s.layer = layer; s.macs = 0; s.bytes = 0;
    for (cudaEvent_t* e : {&s.a, &s.b}) {
        if (!event_pool.empty()) { *e = event_pool.back(); event_pool.pop_back(); }
        else cudaEventCreate(e);
    }
    // inside a stream capture the record becomes an EXTERNAL event node: it fires at every replay of the graph
    if (prof_capturing) cudaEventRecordWithFlags(s.a, st, cudaEventRecordExternal);
    else cudaEventRecord(s.a, st);
    spans.push_back(s);
}
void Engine::prof_end(cudaStream_t st) {
    if (!profiling || spans.empty() || (profiling == 2 && !prof_capturing)) return;
    if (prof_capturing) cudaEventRecordWithFlags(spans.back().b, st, cudaEventRecordExternal);
    else cudaEventRecord(spans.back().b, st);
}
void Engine::prof_note(double macs, double bytes) {
    if (!profiling || spans.empty() || (profiling == 2 && !prof_capturing)) return;
    spans.back().macs += macs; spans.back().bytes += bytes;
}
int Engine::prof_fold(std::vector<Span>& v, bool recycle) {
    // an EMPTY span (two back-to-back event records, cat < 0) calibrates what the event nodes themselves cost inside a
    // graph; it is subtracted from every span of the same replay
    float t0 = 0.f;
    for (auto& s : v)
        if (s.cat < 0) {
            MS_CHECK_CUDA(cudaEventSynchronize(s.b));
            MS_CHECK_CUDA(cudaEventElapsedTime(&t0, s.a, s.b));
            prof_event_overhead_ms = t0;
        }
    for (auto& s : v) {
        if (s.cat < 0) { if (recycle) { event_pool.push_back(s.a); event_pool.push_back(s.b); } continue; }
        MS_CHECK_CUDA(cudaEventSynchronize(s.b));
        float ms = 0.f;
        MS_CHECK_CUDA(cudaEventElapsedTime(&ms, s.a, s.b));
        ms = ms > t0 ? ms - t0 : 0.f;
        cat_ms[s.cat] += ms; cat_calls[s.cat] += 1; cat_macs[s.cat] += s.macs; cat_bytes[s.cat] += s.bytes;
        if (s.layer >= 0 && s.cat <= CAT_CONV_WGRAD && s.layer < (int)layer_ms[s.cat].size()) {
            layer_ms[s.cat][s.layer] += ms; layer_calls[s.cat][s.layer] += 1;
        }
        if (recycle) { event_pool.push_back(s.a); event_pool.push_back(s.b); }
    }
    if (recycle) v.clear();
    return 0;
}
int Engine::prof_collect() { return prof_fold(spans, true); }

int Engine::build_madnet() {
    layers.clear();
    char buf[128];
    for (int i = 1; i <= 12; ++i) {
        ConvLayer L;
        snprintf(buf, sizeof buf, "left/conv%d", i); L.name = buf;
        snprintf(buf, sizeof buf, "model/gc-read-pyramid/conv%d", i); L.scope = buf;
        L.bname = "biases";
        L.kh = L.kw = 3; L.cin = PYR_CH[i - 1]; L.cout = PYR_CH[i]; L.stride = (i % 2) ? 2 : 1; L.dil = 1;
        L.alpha = MAD_ALPHA; L.transposed = 0; L.group = -1; L.w_off = L.b_off = 0;
        layers.push_back(L);
    }
    const int nd = (2 * radius_d) / corr_stride + 1;
    for (int k = 6; k >= 2; --k) {
        int cin = PYR_CH[feat_of(k)] + nd + (k < 6 ? 1 : 0);
        for (int j = 1; j <= 6; ++j) {
            ConvLayer L;
            snprintf(buf, sizeof buf, "fgc-volume-filtering-%d/disp%d", k, j); L.name = buf;
            snprintf(buf, sizeof buf, "model/G%d/fgc-volume-filtering-%d/disp-%d", k, k, j); L.scope = buf;
            L.bname = "biases";
            L.kh = L.kw = 3; L.cin = cin; L.cout = EST_CH[j - 1]; L.stride = 1; L.dil = 1;
            L.alpha = j < 6 ? MAD_ALPHA : 1.f; L.transposed = 0; L.group = -1; L.w_off = L.b_off = 0;
            layers.push_back(L);
            cin = L.cout;
        }
    }
    int cin = PYR_CH[4] + 1;
    for (int j = 1; j <= 7; ++j) {
        ConvLayer L;
        snprintf(buf, sizeof buf, "context%d", j); L.name = buf;
        snprintf(buf, sizeof buf, "model/context-%d", j); L.scope = buf;
        L.bname = "biases";
        L.kh = L.kw = 3; L.cin = cin; L.cout = CTX_CH[j - 1]; L.stride = 1; L.dil = CTX_RATE[j - 1];
        L.alpha = j < 7 ? MAD_ALPHA : 1.f; L.transposed = 0; L.group = -1; L.w_off = L.b_off = 0;
        layers.push_back(L);
        cin = L.cout;
    }
    return 0;
}

int Engine::finalize_groups(const int* group_of_layer, int ng) {
    n_groups = ng;
    for (size_t i = 0; i < layers.size(); ++i) {
        int g = group_of_layer ? group_of_layer[i] : -1;
        MS_REQUIRE(g >= -1 && g < ng, "finalize_groups: group index out of range");
        layers[i].group = g;
    }
    group_begin.assign(ng, 0);
    group_end.assign(ng, 0);
    size_t off = 0;
    auto place = [&](ConvLayer& L) {
        L.w_off = off; off += (size_t)L.kh * L.kw * L.cin * L.cout; off = (off + 3) / 4 * 4;
        L.b_off = off; off += (size_t)L.cout; off = (off + 3) / 4 * 4;
    };
    for (int g = 0; g < ng; ++g) {
        group_begin[g] = off;
        for (auto& L : layers) if (L.group == g) place(L);
        group_end[g] = off;
    }
    for (auto& L : layers) if (L.group < 0) place(L);
    n_params = off;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// workspace layout
// ---------------------------------------------------------------------------------------------
void Engine::plan_views(int li, const TView& x, const TView& y, const TView& dpre, const TView& dx) {
    plan[li] = ConvPlan{};
    plan[li].x = x; plan[li].y = y; plan[li].dpre = dpre; plan[li].dx = dx;
}

// Every layer's kernels, in order of preference, from the views plan_views() recorded; then what they read: weight
// tiles and prep jobs of BF forwards and dgrads, fp16 planes of BF forward inputs, bf16 planes of the output gradients
// of BF dgrads and weight gradients, and the sizes of the weight-gradient workspace, its re-split scratch planes and
// the transposed-weight scratch.  -2: a layer's views do not fit it.
int Engine::plan_convs(Bump& A, size_t& max_wg, size_t& max_wt) {
    wg_xp_halfs = 0;
    for (size_t li = 0; li < layers.size(); ++li) {
        const ConvLayer& L = layers[li];
        ConvPlan& P = plan[li];
        ConvGemm f, d;
        ConvWgrad q;
        MS_REQUIRE(fwd_args((int)li, f) && wgrad_args((int)li, q) && (!P.dx.p || dgrad_args((int)li, d)),
                   "layer " + std::to_string(li) + " (" + L.name + "): its planned views do not fit it");
        if (conv_head_kind(f) == 1) P.fwd = ConvPlan::FWD_HEAD;
        else if (conv_one_channel_supported(f)) P.fwd = ConvPlan::FWD_ONE_CHANNEL;
        else if (!L.transposed && conv_stem_fwd_supported(f)) P.fwd = ConvPlan::FWD_STEM;
        // the 16-channel full-resolution layers (conv2: 2 x 192 x 640 x 16) would fill one eighth of the swap-AB tile's
        // accumulator rows; the shared-memory tiled direct kernel is bandwidth-shaped
        else if (!L.transposed && conv_small_fwd_supported(f)) P.fwd = ConvPlan::FWD_SMALL;
        else if (conv_bf_supported(f)) P.fwd = ConvPlan::FWD_BF;
        else P.fwd = ConvPlan::FWD_GEMM;
        // (an unaligned channel slice -- DispNet conv_redir's output gradient, channel 81 of gd_cat3 -- gets no planes:
        //  its dgrad and weight gradient stay in fp32)
        const bool dpre_planes = (reinterpret_cast<uintptr_t>(P.dpre.p) & 15) == 0;
        P.dgrad = ConvPlan::DGRAD_GEMM;
        if (P.dx.p) {
            if (conv_head_kind(d) == 2) P.dgrad = ConvPlan::DGRAD_HEAD;
            else if (dpre_planes && conv_bf_supported(d)) P.dgrad = ConvPlan::DGRAD_BF;
        }
        // the image has no tensor-core weight gradient (MADNet conv1: conv_small_wgrad)
        if (conv_stem_wgrad_supported(q)) P.wgrad = ConvPlan::WGRAD_STEM;
        else if (P.x.p != img.p && dpre_planes && wgrad_bf_supported(q)) P.wgrad = ConvPlan::WGRAD_BF;
        else if (conv_head_wgrad_supported(q)) P.wgrad = ConvPlan::WGRAD_HEAD;
        else P.wgrad = ConvPlan::WGRAD_FP32;

        const int taps = L.kh * L.kw;
        size_t wg;
        switch (P.wgrad) {
        case ConvPlan::WGRAD_BF:    // wgrad_bf fits its split count to the workspace: 48 Mi floats bound the widest layers
            wg = std::min<size_t>(wgrad_bf_workspace_floats(L.kh, L.kw, q.x.c, q.dy.c), (size_t)48 << 20);
            wg_xp_halfs = std::max(wg_xp_halfs, P.x.pixels() * (size_t)((P.x.c + 7) / 8 * 8));
            break;
        case ConvPlan::WGRAD_STEM: wg = conv_stem_wgrad_workspace_floats(q); break;
        case ConvPlan::WGRAD_HEAD: wg = conv_head_wgrad_workspace_floats(q); break;
        default: wg = conv_wgrad_workspace_floats(taps, q.x.c, q.dy.c, q.dy.pixels());
        }
        if (L.transposed) wg = std::max(wg, (size_t)128 * L.cout);          // + bias_grad's partials (<= 128 blocks)
        max_wg = std::max(max_wg, wg);
        max_wt = std::max(max_wt, (size_t)taps * L.cin * L.cout);
        if (P.fwd == ConvPlan::FWD_BF) planes[P.x.p] = ActPlanes{nullptr, nullptr, (P.x.c + 7) / 8 * 8, 1, 1.f};
        if (P.dgrad == ConvPlan::DGRAD_BF || P.wgrad == ConvPlan::WGRAD_BF) planes[P.dpre.p] = ActPlanes{nullptr, nullptr, (P.dpre.c + 7) / 8 * 8, 0, 1.f};
    }
    // a tensor's planes cover the widest view any layer runs on (d_c2: conv2's output, conv_redir reads its left half)
    std::map<const float*, size_t> pixels;
    for (const ConvPlan& P : plan)
        for (const TView* v : {&P.x, &P.y, &P.dpre, &P.dx})
            if (planes.count(v->p)) pixels[v->p] = std::max(pixels[v->p], v->pixels());
    for (auto& e : planes) {
        ActPlanes& pl = e.second;
        pl.scale = pl.fmt == 1 ? act_scale : 1.f;
        pl.hi = A.alloc((pixels[e.first] * pl.cs + 1) / 2);           // 16-bit elements -> floats
        pl.lo = A.alloc((pixels[e.first] * pl.cs + 1) / 2);
    }
    auto planes_of = [&](const TView& v) -> const ActPlanes* { auto it = planes.find(v.p); return it == planes.end() ? nullptr : &it->second; };
    for (ConvPlan& P : plan) { P.xp = planes_of(P.x); P.yp = planes_of(P.y); P.dp = planes_of(P.dpre); P.dxp = planes_of(P.dx); }
    // split 16-bit weight tiles of the BF directions (forward: fp16, dgrad: bf16), with their prep jobs grouped by MAD
    // module so that an update refreshes exactly the tiles of the weights it moved
    bf_jobs.clear(); bf_job_begin.assign(n_groups + 1, 0); bf_job_end.assign(n_groups + 1, 0);
    bf_max_total = 0;
    for (int gidx = 0; gidx <= n_groups; ++gidx) {
        bf_job_begin[gidx] = (int)bf_jobs.size();
        for (size_t li = 0; li < layers.size(); ++li) {
            const ConvLayer& L = layers[li];
            ConvPlan& P = plan[li];
            if ((L.group < 0 ? n_groups : L.group) != gidx) continue;
            for (int dir = 0; dir < 2; ++dir) {
                if (dir == 0 ? P.fwd != ConvPlan::FWD_BF : P.dgrad != ConvPlan::DGRAD_BF) continue;
                // forward: M = cout, K = cin; dgrad: M = cin, K = cout.  Canonical W is [tap][cin][cout] ([tap][cout][cin]
                // for a transposed layer)
                const int M = dir == 0 ? L.cout : L.cin, K = dir == 0 ? L.cin : L.cout;
                int Mpad, Kpad; conv_bf_weight_dims(M, K, Mpad, Kpad);
                const size_t halfs = conv_bf_weight_halfs(L.kh * L.kw, M, K);
                P.tiles[dir] = A.alloc((halfs + 1) / 2);
                bf_jobs.push_back(BfPrepJob{Wt ? Wt + L.w_off : nullptr, P.tiles[dir], L.kh * L.kw, M, K, Mpad, Kpad,
                                            (dir == 0) != (L.transposed != 0), dir == 0 ? 1 : 0});
                bf_max_total = std::max(bf_max_total, halfs);
            }
        }
        bf_job_end[gidx] = (int)bf_jobs.size();
    }
    return 0;
}

int Engine::layout(float* base, size_t* floats) {
    *floats = 0;
    // the sizing pass lays out against a stand-in base with the workspace's 256-byte alignment (never dereferenced), so
    // that both passes plan from the same views
    Bump A{base ? base : reinterpret_cast<float*>(uintptr_t{256}), 0};
    auto alloc = [&](size_t n) -> float* { return A.alloc(n); };
    auto tens = [&](int n, int h, int w, int c, int cs = 0) { return A.tens(n, h, w, c, cs); };
    tensors.clear();
    planes.clear(); fresh.clear();
    plan.assign(layers.size(), ConvPlan{});
    char nm[128];
    const int nd = (2 * radius_d) / corr_stride + 1;
    TView raw_l = tens(B, H, W, 3), raw_r = tens(B, H, W, 3);
    tensors["raw_left"] = raw_l; tensors["raw_right"] = raw_r;
    img = tens(2 * B, Hp, Wp, 3, 4);
    tensors["img"] = img;
    if (net == 1) {
        layout_dispnet(A);
    } else {
    int h = Hp, w = Wp;
    for (int i = 1; i <= 12; ++i) {
        if (i % 2) { h = (h + 1) / 2; w = (w + 1) / 2; }
        pyr[i] = tens(2 * B, h, w, PYR_CH[i]);
        g_pyr[i] = tens(2 * B, h, w, PYR_CH[i]);
        plan_views(i - 1, i > 1 ? pyr[i - 1] : img, pyr[i], g_pyr[i], i > 1 ? g_pyr[i - 1] : TView{});
        snprintf(nm, sizeof nm, "left/conv%d", i); tensors[nm] = batch(pyr[i], 0, B);
        snprintf(nm, sizeof nm, "right/conv%d", i); tensors[nm] = batch(pyr[i], B, B);
        snprintf(nm, sizeof nm, "grad/left/conv%d", i); tensors[nm] = batch(g_pyr[i], 0, B);
        snprintf(nm, sizeof nm, "grad/right/conv%d", i); tensors[nm] = batch(g_pyr[i], B, B);
    }
    ctxin = tens(B, pyr[4].h, pyr[4].w, PYR_CH[4] + 1, pad4(PYR_CH[4] + 1));
    g_ctxin = tens(B, pyr[4].h, pyr[4].w, PYR_CH[4] + 1, pad4(PYR_CH[4] + 1));
    tensors["ctxin"] = ctxin; tensors["grad/ctxin"] = g_ctxin;
    for (int k = 6; k >= 2; --k) {
        const int f = feat_of(k), C = PYR_CH[f];
        const int hh = pyr[f].h, ww = pyr[f].w;
        const int ct = C + nd + (k < 6 ? 1 : 0);
        cost[k] = tens(B, hh, ww, ct, pad4(ct));
        g_cost[k] = tens(B, hh, ww, ct, pad4(ct));
        snprintf(nm, sizeof nm, "cost%d", k); tensors[nm] = cost[k];
        snprintf(nm, sizeof nm, "grad/cost%d", k); tensors[nm] = g_cost[k];
        for (int j = 1; j <= 5; ++j) {
            est[k][j] = tens(B, hh, ww, EST_CH[j - 1]);
            g_est[k][j] = tens(B, hh, ww, EST_CH[j - 1]);
            snprintf(nm, sizeof nm, "fgc-volume-filtering-%d/disp%d", k, j); tensors[nm] = est[k][j];
            snprintf(nm, sizeof nm, "grad/fgc-volume-filtering-%d/disp%d", k, j); tensors[nm] = g_est[k][j];
        }
        if (k == 2) V[k] = slice(ctxin, PYR_CH[4], 1);
        else V[k] = tens(B, hh, ww, 1);
        g_V[k] = tens(B, hh, ww, 1);
        g_u[k] = tens(B, hh, ww, 1);
        snprintf(nm, sizeof nm, "fgc-volume-filtering-%d/disp6", k); tensors[nm] = V[k];
        snprintf(nm, sizeof nm, "grad/fgc-volume-filtering-%d/disp6", k); tensors[nm] = g_V[k];
        snprintf(nm, sizeof nm, "grad/u%d", k); tensors[nm] = g_u[k];
        for (int j = 1; j <= 6; ++j)
            plan_views(est_layer(k, j), j > 1 ? est[k][j - 1] : cost[k], j < 6 ? est[k][j] : V[k], j < 6 ? g_est[k][j] : g_V[k],
                       j > 1 ? g_est[k][j - 1] : g_cost[k]);
    }
    for (int j = 1; j <= 6; ++j) {
        ctx[j] = tens(B, pyr[4].h, pyr[4].w, CTX_CH[j - 1]);
        g_ctx[j] = tens(B, pyr[4].h, pyr[4].w, CTX_CH[j - 1]);
        snprintf(nm, sizeof nm, "context%d", j); tensors[nm] = ctx[j];
        snprintf(nm, sizeof nm, "grad/context%d", j); tensors[nm] = g_ctx[j];
    }
    final_ = tens(B, pyr[4].h, pyr[4].w, 1);
    g_final = tens(B, pyr[4].h, pyr[4].w, 1);
    tensors["final_disp"] = final_; tensors["grad/final_disp"] = g_final;
    for (int j = 1; j <= 7; ++j)
        plan_views(ctx_layer(j), j > 1 ? ctx[j - 1] : ctxin, j < 7 ? ctx[j] : final_, j < 7 ? g_ctx[j] : g_final,
                   j > 1 ? g_ctx[j - 1] : g_ctxin);
    }   // net == 0
    n_disp = net == 1 ? 7 : 6;
    for (int i = 0; i < n_disp; ++i) {
        disp[i] = tens(B, H, W, 1);
        snprintf(nm, sizeof nm, "disp%d", i); tensors[nm] = disp[i];
    }
    tensors["rescaled_prediction"] = disp[n_disp - 1];
    g_disp = tens(B, H, W, 1);
    tensors["grad/disp"] = g_disp;
    size_t max_wg = 0, max_wt = 0;
    if (plan_convs(A, max_wg, max_wt)) return -2;
    wT_floats = max_wt; wT = alloc(max_wt);
    wg_ws_floats = max_wg; wg_ws = alloc(max_wg);
    if (wg_xp_halfs) {
        wg_xp.hi = alloc((wg_xp_halfs + 1) / 2); wg_xp.lo = alloc((wg_xp_halfs + 1) / 2); wg_xp.fmt = 0;
    }
    splitk[0].bf_part = alloc(conv_bf_part_floats());
    splitk[0].bf_tickets = reinterpret_cast<unsigned int*>(alloc(conv_bf_ticket_words()));
    bf_jobs_dev = reinterpret_cast<BfPrepJob*>(alloc((bf_jobs.size() + 1) * sizeof(BfPrepJob) / sizeof(float) + 16));
    splitk[0].gemm_part = alloc(conv_gemm_part_floats());
    rs_tmp_floats = (size_t)B * H * Wp; rs_tmp = alloc(rs_tmp_floats);
    loss_ws_floats = loss_workspace_floats(B, H, W); loss_ws = alloc(loss_ws_floats);
    scalars = alloc(64);
    u8_stage = reinterpret_cast<unsigned char*>(alloc((2 * u8_stage_right_offset((size_t)B * H * W * 3)) / 4 + 64));
    gt = alloc((size_t)B * H * W);
    proxy = alloc((size_t)B * H * W);
    // what a MAD train op on its branch (mad_branch) shares with the forward's tail: the split-K scratch of its dgrads
    // and the loss workspace.  Its own copies; everything else it writes (g_*, Gr, Mo, wg_ws, wg_xp, rs_tmp, g_disp, the
    // module's weights and tiles, scalars[1]) no later forward kernel touches, and the tail runs no conv on wT
    splitk[1] = splitk[0];
    loss_full_ws = nullptr;
    if (net == 0 && n_groups > 0) {
        splitk[1].bf_part = alloc(conv_bf_part_floats());
        splitk[1].bf_tickets = reinterpret_cast<unsigned int*>(alloc(conv_bf_ticket_words()));
        bool module_gemm = false;
        for (size_t li = 0; li < layers.size(); ++li)
            module_gemm |= layers[li].group >= 0 && plan[li].dx.p && plan[li].dgrad == ConvPlan::DGRAD_GEMM;
        if (module_gemm) splitk[1].gemm_part = alloc(conv_gemm_part_floats());
        loss_full_ws = alloc(loss_value_workspace_floats(B, H, W));
    }
    *floats = A.off;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// conv helpers
// ---------------------------------------------------------------------------------------------
// (every *_args call below fits: plan_convs checked each layer's views at layout time)
int Engine::conv_fwd(int li, const float* res, int res_cs, cudaStream_t st) {
    const ConvLayer& L = layers[li];
    const ConvPlan& P = plan[li];
    ConvGemm p;
    fwd_args(li, p);
    p.res = res; p.res_cs = res_cs;
    if (L.transposed && P.fwd != ConvPlan::FWD_BF && transpose_taps(Wt + L.w_off, wT, L.kh * L.kw, L.cout, L.cin, st)) return -1;
    prof_begin(CAT_CONV_FWD, st, li);
    int rc;
    switch (P.fwd) {
    case ConvPlan::FWD_HEAD: rc = conv_head(p, st); break;
    case ConvPlan::FWD_ONE_CHANNEL:
        p.wmat = Wt + L.w_off;                       // [tap][1][1]: canonical weights serve either orientation
        rc = conv_one_channel(p, st);
        break;
    case ConvPlan::FWD_STEM: rc = conv_stem_fwd(p, P.yp, st); break;
    case ConvPlan::FWD_SMALL: rc = conv_small_fwd(p, st); break;
    case ConvPlan::FWD_BF:
        rc = ensure_planes(P.x, P.xp, st);
        if (!rc) rc = conv_bf(p, *P.xp, P.tiles[0], P.yp, sk().bf_part, sk().bf_tickets, st);
        break;
    default: rc = conv_gemm(p, st);
    }
    planes_written(P.y, P.yp, P.fwd == ConvPlan::FWD_STEM || P.fwd == ConvPlan::FWD_BF);
    prof_end(st);
    prof_note((double)P.y.pixels() * L.kh * L.kw * L.cin * L.cout / (L.transposed ? L.stride * L.stride : 1), 0);
    return rc;
}

// weight gradient of a planned layer on stream st
int Engine::wgrad(const ConvLayer& L, const ConvPlan& P, const ConvWgrad& q, cudaStream_t st) {
    switch (P.wgrad) {
    case ConvPlan::WGRAD_BF: {
        // bf16 copy of the forward input in scratch planes: a wgmma takes one 16-bit element type for both operands, so
        // the fp16 forward planes cannot pair with the bf16 gradient planes
        ActPlanes xb = wg_xp; xb.cs = (P.x.c + 7) / 8 * 8;
        MS_REQUIRE(P.x.pixels() * (size_t)xb.cs <= wg_xp_halfs, "wgrad: scratch planes too small");
        if (split_planes(P.x, xb, st)) return -1;
        return L.transposed ? wgrad_bf(q, *P.dp, xb, st) : wgrad_bf(q, xb, *P.dp, st);
    }
    case ConvPlan::WGRAD_STEM: return conv_stem_wgrad(q, st);           // DispNet conv1
    case ConvPlan::WGRAD_HEAD: return conv_head_wgrad(q, st);           // single-channel heads, up_predict
    default: return conv_wgrad(q, st);
    }
}

// from the planned output gradient P.dpre (wrt the pre-activation output): the weight gradient (want_wgrad) and the
// input gradient into P.dx (want_dx; dx_acc: added to P.dx; dx_slope != 1: masked by the leaky ReLU of P.x, that slope)
int Engine::conv_bwd(int li, int want_dx, float dx_slope, int dx_acc, int want_wgrad, cudaStream_t st) {
    const ConvLayer& L = layers[li];
    const ConvPlan& P = plan[li];
    MS_REQUIRE(!L.transposed, "conv_bwd: transposed layers use deconv_bwd");
    MS_REQUIRE(!want_dx || P.dx.p, "conv_bwd: layer " + L.name + " has no planned input gradient");
    ConvWgrad q;
    ConvGemm p;
    wgrad_args(li, q);
    if (want_dx) dgrad_args(li, p);
    if (net == 1) fresh.clear();    // DispNet's backward mutates gradient tensors in place between convs: always re-split
    if (want_wgrad) {
        prof_begin(CAT_CONV_WGRAD, st, li);
        // the planes of dpre also feed the dgrad below: they are produced on `st` BEFORE the fork
        int rc = P.wgrad == ConvPlan::WGRAD_BF ? ensure_planes(P.dpre, P.dp, st) : 0;
        cudaStream_t ws = st;
        if (!rc) rc = fork_wgrad(st, &ws);
        if (!rc) rc = wgrad(L, P, q, ws);
        prof_end(st);
        prof_note((double)P.dpre.pixels() * L.kh * L.kw * L.cin * L.cout, 0);
        if (rc) return -1;
    }
    if (want_dx) {
        if (dx_slope != 1.f) { p.mask = P.x.p; p.mask_cs = P.x.cs; p.mask_alpha = dx_slope; }
        p.accumulate = dx_acc;
        prof_begin(CAT_CONV_DGRAD, st, li);
        int rc;
        switch (P.dgrad) {
        case ConvPlan::DGRAD_HEAD: rc = conv_head(p, st); break;    // [tap][cin][1] == [tap][1][cin]: canonical weights
        case ConvPlan::DGRAD_BF:
            rc = ensure_planes(P.dpre, P.dp, st);
            if (!rc) rc = conv_bf(p, *P.dp, P.tiles[1], P.dxp, sk().bf_part, sk().bf_tickets, st);
            break;
        default:
            p.wmat = wT;
            rc = transpose_taps(Wt + L.w_off, wT, L.kh * L.kw, L.cin, L.cout, st);   // -> [tap][cout][cin]
            if (!rc) rc = conv_gemm(p, st);
        }
        planes_written(P.dx, P.dxp, P.dgrad == ConvPlan::DGRAD_BF);
        prof_end(st);
        prof_note((double)P.dpre.pixels() * L.kh * L.kw * L.cin * L.cout, 0);
        if (rc) return -1;
    }
    return 0;
}

bool Engine::trainable(int layer, int mode, int group) const {
    if (mode == 2) return true;
    if (mode == 1) return layers[layer].group == group;
    return false;
}

// ---------------------------------------------------------------------------------------------
// input / forward
// ---------------------------------------------------------------------------------------------
int Engine::set_input(const float* left, const float* right, cudaStream_t st) {
    MS_REQUIRE(bound, "engine not bound");
    TView rl = tensors["raw_left"], rr = tensors["raw_right"];
    size_t bytes = (size_t)B * H * W * 3 * sizeof(float);
    MS_CHECK_CUDA(cudaMemcpyAsync(rl.p, left, bytes, cudaMemcpyDefault, st));
    MS_CHECK_CUDA(cudaMemcpyAsync(rr.p, right, bytes, cudaMemcpyDefault, st));
    rs_fresh = false;
    return 0;
}

// uint8 frames (host or device): 4x fewer bytes over PCIe than fp32; converted on the device.  Any B*H*W: the right frame
// is staged at the next 4-byte boundary so that both halves are read with aligned uchar4 loads.
int Engine::set_input_u8(const unsigned char* left, const unsigned char* right, cudaStream_t st) {
    MS_REQUIRE(bound, "engine not bound");
    TView rl = tensors["raw_left"], rr = tensors["raw_right"];
    const size_t n = (size_t)B * H * W * 3;
    unsigned char* right_stage = u8_stage + u8_stage_right_offset(n);
    MS_CHECK_CUDA(cudaMemcpyAsync(u8_stage, left, n, cudaMemcpyDefault, st));
    MS_CHECK_CUDA(cudaMemcpyAsync(right_stage, right, n, cudaMemcpyDefault, st));
    rs_fresh = false;
    if (u8_to_f32(u8_stage, rl.p, n, st)) return -1;
    return u8_to_f32(right_stage, rr.p, n, st);
}

// uint8 device frames [B,h,w,3] at camera size: rescale to (rh, rw) and centre crop / zero pad to (H, W) in one pass;
// with rectification set, the frames are first rectified into the scratch and the rescale reads them from there
int Engine::set_input_u8_resized(const unsigned char* left, const unsigned char* right, int h, int w, int rh, int rw,
                                 cudaStream_t st) {
    MS_REQUIRE(bound, "engine not bound");
    rs_fresh = false;
    if (rect_map_l) {
        MS_REQUIRE(h == rect_h && w == rect_w, "set_input_u8_resized: frames are " + std::to_string(h) + "x" + std::to_string(w) +
                                               ", the rectification tables " + std::to_string(rect_h) + "x" + std::to_string(rect_w));
        unsigned char* rl = rect_scratch;
        unsigned char* rr = rect_scratch + (size_t)B * h * w * 3;
        if (rectify_u8(left, right, rect_map_l, rect_map_r, B, h, w, rl, rr, st)) return -1;
        left = rl; right = rr;
    }
    return u8_resize_crop(left, right, B, h, w, rh, rw, tensors["raw_left"].p, tensors["raw_right"].p, H, W, st);
}

int Engine::set_rectification(const float* map_left, const float* map_right, int h, int w, unsigned char* scratch,
                              size_t scratch_bytes) {
    if (!map_left && !map_right) {
        rect_map_l = rect_map_r = nullptr; rect_h = rect_w = 0; rect_scratch = nullptr;
        return 0;
    }
    MS_REQUIRE(map_left && map_right, "set_rectification: both cameras need a table (two NULL tables turn it off)");
    MS_REQUIRE(h >= 1 && w >= 1, "set_rectification: bad table size");
    MS_REQUIRE(((reinterpret_cast<uintptr_t>(map_left) | reinterpret_cast<uintptr_t>(map_right)) & 7) == 0,
               "set_rectification: tables must be 8-byte aligned");
    const size_t need = 2 * (size_t)B * h * w * 3;
    MS_REQUIRE(scratch && scratch_bytes >= need,
               "set_rectification: the scratch must hold both rectified frames (" + std::to_string(need) + " bytes)");
    rect_map_l = map_left; rect_map_r = map_right; rect_h = h; rect_w = w; rect_scratch = scratch;
    return 0;
}

// The scratch of module losses at 1/s resolution: left_s, right_s, proxy_s, the module disparity at loss resolution, then
// per module (source V[6-g], or final_ for module 4) the tap tables of rs_disp.  base == nullptr: sizing only.
size_t Engine::rs_layout(int s, float* base) {
    Bump A{base ? base : reinterpret_cast<float*>(uintptr_t{256}), 0};
    const int h = H / s, w = W / s;
    TView l = A.tens(B, h, w, 3), r = A.tens(B, h, w, 3), p = A.tens(B, h, w, 1), d = A.tens(B, h, w, 1);
    RsTables t[5];
    for (int g = 0; g < 5; ++g) {
        const TView& src = g < 4 ? V[6 - g] : final_;
        t[g].rows = reinterpret_cast<RsTap*>(A.alloc((size_t)h * sizeof(RsTap) / sizeof(float)));
        t[g].cols = reinterpret_cast<RsTap*>(A.alloc((size_t)w * sizeof(RsTap) / sizeof(float)));
        t[g].rrange = reinterpret_cast<RsRange*>(A.alloc((size_t)src.h * sizeof(RsRange) / sizeof(float)));
        t[g].crange = reinterpret_cast<RsRange*>(A.alloc((size_t)src.w * sizeof(RsRange) / sizeof(float)));
    }
    if (base) {
        rs_left = l; rs_right = r; rs_proxy = p; rs_disp = d;
        for (int g = 0; g < 5; ++g) rs_tab[g] = t[g];
    }
    return A.off;
}

int Engine::reprojection_scratch_floats(int s, size_t* floats) {
    *floats = 0;
    MS_REQUIRE(s >= 1, "reprojection scale must be >= 1, got " + std::to_string(s));
    if (s == 1) return 0;
    // the reference asserts one train op per side output, which DispNet does not have (Stereo_Online_Adaptation.py:97)
    MS_REQUIRE(net == 0, "reprojection scale " + std::to_string(s) + ": only MADNet has MAD train ops (DispNet: scale 1)");
    MS_REQUIRE(bound, "reprojection scale: engine not bound");
    MS_REQUIRE(H / s >= 3 && W / s >= 3, "reprojection scale " + std::to_string(s) + ": the loss resolution " +
                                         std::to_string(H / s) + "x" + std::to_string(W / s) + " is below the 3x3 SSIM window");
    *floats = rs_layout(s, nullptr);
    return 0;
}

int Engine::set_reprojection_scale(int s, float* scratch, size_t scratch_floats) {
    size_t need = 0;
    if (s == 1 || (s > 1 && !scratch)) {        // back to full-resolution module losses
        if (rs_scale != 1) drop_graphs();
        rs_scale = 1; rs_fresh = false;
        for (const char* n : {"rs_left", "rs_right", "rs_proxy", "rs_disp"}) tensors.erase(n);
        return 0;
    }
    if (reprojection_scratch_floats(s, &need)) return -2;
    MS_REQUIRE(scratch_floats >= need, "set_reprojection_scale: the scratch holds " + std::to_string(scratch_floats) +
                                       " floats, scale " + std::to_string(s) + " needs " + std::to_string(need));
    MS_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "set_reprojection_scale: the scratch must be 16B aligned");
    const int h = H / s, w = W / s;
    std::vector<RsTap> rows(h), cols(w);
    std::vector<RsRange> rr, cr;
    MS_CHECK_CUDA(cudaDeviceSynchronize());     // a step in flight may still read the tables being replaced
    rs_layout(s, scratch);
    for (int g = 0; g < 5; ++g) {
        const TView& src = g < 4 ? V[6 - g] : final_;
        rr.resize(src.h); cr.resize(src.w);
        rs_axis_taps(src.h, Hp, H, h, rows.data(), rr.data());
        rs_axis_taps(src.w, Wp, W, w, cols.data(), cr.data());
        MS_CHECK_CUDA(cudaMemcpy(rs_tab[g].rows, rows.data(), rows.size() * sizeof(RsTap), cudaMemcpyHostToDevice));
        MS_CHECK_CUDA(cudaMemcpy(rs_tab[g].cols, cols.data(), cols.size() * sizeof(RsTap), cudaMemcpyHostToDevice));
        MS_CHECK_CUDA(cudaMemcpy(rs_tab[g].rrange, rr.data(), rr.size() * sizeof(RsRange), cudaMemcpyHostToDevice));
        MS_CHECK_CUDA(cudaMemcpy(rs_tab[g].crange, cr.data(), cr.size() * sizeof(RsRange), cudaMemcpyHostToDevice));
    }
    drop_graphs();                              // the loss-resolution kernels and buffers are baked into the step graphs
    rs_scale = s; rs_fresh = false;
    tensors["rs_left"] = rs_left; tensors["rs_right"] = rs_right; tensors["rs_proxy"] = rs_proxy; tensors["rs_disp"] = rs_disp;
    return 0;
}

// left_s, right_s (and proxy_s under the proxy loss) of the current frame
int Engine::rs_prepare_inputs(cudaStream_t st) {
    const bool px = loss_kind == 1;
    if (rs_inputs(tensors["raw_left"].p, tensors["raw_right"].p, px ? proxy : nullptr, B, H, W, rs_left.p, rs_right.p,
                  px ? rs_proxy.p : nullptr, rs_left.h, rs_left.w, rs_scale, st)) return -1;
    rs_fresh = true;
    return 0;
}

int Engine::prep_layers(int group, cudaStream_t st) {
    if (bf_jobs.empty()) return 0;
    int b, e;
    if (group < 0) { b = 0; e = (int)bf_jobs.size(); }
    else { b = bf_job_begin[group]; e = bf_job_end[group]; }
    return bf_prep_weights(bf_jobs_dev + b, e - b, bf_max_total, st);
}

int Engine::forward(int disp_mask, cudaStream_t st, int fork_group, cudaStream_t branch) {
    MS_REQUIRE(bound, "engine not bound");
    MS_REQUIRE(!branch || (net == 0 && fork_group >= 0 && fork_group <= 4), "forward: bad branch point");
    auto fork = [&]() -> int {
        MS_CHECK_CUDA(cudaEventRecord(ev_bfork, st));
        MS_CHECK_CUDA(cudaStreamWaitEvent(branch, ev_bfork, 0));
        return 0;
    };
    fresh.clear();
    const int nd = (2 * radius_d) / corr_stride + 1;
    {
        TView rl = tensors["raw_left"], rr = tensors["raw_right"];
        TView il = batch(img, 0, B), ir = batch(img, B, B);
        // DispNet normalises (x/255 - 100/255, Nets/DispNet.py:59-73); MADNet feeds raw 0..255 (Nets/MadNet.py:56-66)
        const float sc = net == 1 ? 1.f / 255.f : 1.f, bi = net == 1 ? -100.f / 255.f : 0.f;
        if (pad_reflect(rl.p, B, H, W, 3, il.p, Hp, Wp, img.cs, sc, bi, st)) return -1;
        if (pad_reflect(rr.p, B, H, W, 3, ir.p, Hp, Wp, img.cs, sc, bi, st)) return -1;
    }
    if (weights_dirty) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cs);
        MS_REQUIRE(cs == cudaStreamCaptureStatusNone, "forward: weights changed while capturing a graph");
        if (prep_layers(-1, st)) return -1;
        weights_dirty = false;
    }
    if (net == 1) return forward_dispnet(disp_mask, st);
    for (int i = 1; i <= 12; ++i)
        if (conv_fwd(i - 1, nullptr, 0, st)) return -1;
    for (int k = 6; k >= 2; --k) {
        const int f = feat_of(k), C = PYR_CH[f];
        TView Lf = batch(pyr[f], 0, B), Rf = batch(pyr[f], B, B);
        const float* u = nullptr;
        if (k < 6) {
            TView us = slice(cost[k], C + nd, 1);
            if (resize_bilinear(V[k + 1].p, V[k + 1].cs, B, V[k + 1].h, V[k + 1].w, us.p, us.cs, cost[k].h, cost[k].w,
                                cost[k].h, cost[k].w, 1.f, 0, 20.f / (float)(1 << k), 0, st)) return -1;
            if (warping) u = us.p;
        }
        CorrFwd cf{};
        cf.left = Lf.p; cf.lcs = Lf.cs; cf.right = Rf.p; cf.rcs = Rf.cs;
        cf.u = u; cf.ucs = cost[k].cs;
        cf.out = cost[k].p; cf.ocs = cost[k].cs;
        cf.out2 = (k == 2) ? ctxin.p : nullptr; cf.o2cs = ctxin.cs;
        cf.B = B; cf.h = cost[k].h; cf.w = cost[k].w; cf.C = C; cf.max_disp = radius_d; cf.stride = corr_stride;
        cf.copy_left = 1; cf.u_chan = (k < 6) ? 1 : 0;
        prof_begin(CAT_CORR_FWD, st);
        int crc = corr_fwd(cf, st);
        prof_end(st);
        prof_note(0, (double)B * cf.h * cf.w * (3.0 * C + nd + (cf.u_chan ? 1 : 0) + (cf.out2 ? C : 0)) * 4.0);   // reads L, R(, u); writes corr + the left copy (fused concat)
        if (crc) return -1;
        for (int j = 1; j <= 6; ++j)
            if (conv_fwd(est_layer(k, j), nullptr, 0, st)) return -1;
        if (branch && fork_group == 6 - k && fork()) return -1;
    }
    for (int j = 1; j <= 7; ++j)
        if (conv_fwd(ctx_layer(j), j == 7 ? V[2].p : nullptr, V[2].cs, st)) return -1;
    if (branch && fork_group == 4 && fork()) return -1;
    for (int i = 0; i < 6; ++i) {
        if (!(disp_mask & (1 << i))) continue;
        const TView& src = (i < 4) ? V[6 - i] : final_;
        cudaStream_t s = branch && i == fork_group ? branch : st;
        if (i < 5) {
            if (resize_bilinear(src.p, src.cs, B, src.h, src.w, disp[i].p, 1, Hp, Wp, H, W, -20.f, 1, 1.f, 0, s)) return -1;
        } else {
            if (resize_bilinear(src.p, src.cs, B, src.h, src.w, disp[i].p, 1, Hp, Wp, H, W, 1.f, 0, -20.f, 1, s)) return -1;
        }
    }
    return 0;
}

int Engine::loss(int which, int with_grad, int slot, float grad_scale, cudaStream_t st) {
    MS_REQUIRE(bound && which >= 0 && which < n_disp && slot >= 0 && slot < 2, "loss: bad arguments");
    // the full-resolution loss of a MAD step runs beside the module's loss (mad_branch): a workspace of its own
    float* ws = slot == 0 && !with_grad && loss_full_ws ? loss_full_ws : loss_ws;
    if (rs_module(which, slot)) {
        // Stereo_Online_Adaptation.py:91-107 / Stereo_Continual_Adaptation.py:95-112 at scale s: the module disparity and
        // the images (proxy) at H/s x W/s.  The reference's multiplier H // p.shape[1] is 1 (its disparities are already
        // full resolution), so the disparity stays in full-resolution pixels: kept as the reference computes it
        if (!rs_fresh && rs_prepare_inputs(st)) return -1;
        const TView& src = which < 4 ? V[6 - which] : final_;
        const int h = rs_disp.h, w = rs_disp.w;
        prof_begin(CAT_LOSS, st);
        int rc = rs_module_disp(src.p, src.cs, B, src.h, src.w, rs_tab[which].rows, rs_tab[which].cols, rs_disp.p, h, w, -20.f, st);
        if (!rc && loss_kind == 1) {
            rc = proxy_loss(rs_disp.p, rs_proxy.p, B * h * w, proxy_w_module, grad_scale, scalars + slot,
                            with_grad ? g_disp.p : nullptr, ws, st);
        } else if (!rc) {
            ReprojLoss p{};
            p.left = rs_left.p; p.right = rs_right.p; p.disp = rs_disp.p; p.loss = scalars + slot;
            p.ddisp = with_grad ? g_disp.p : nullptr;
            p.workspace = ws; p.B = B; p.H = h; p.W = w; p.grad_scale = grad_scale;
            rc = reproj_loss(p, st);
        }
        prof_end(st);
        return rc;
    }
    if (loss_kind == 1) {
        // Stereo_Continual_Adaptation.py:75 (full-resolution loss, weight 0.01; also the FULL train op :133) and :112
        // (module losses, weight 0.1)
        const float wgt = slot == 0 ? proxy_w_full : proxy_w_module;
        prof_begin(CAT_LOSS, st);
        int rc = proxy_loss(disp[which].p, proxy, B * H * W, wgt, grad_scale, scalars + slot, with_grad ? g_disp.p : nullptr, ws, st);
        prof_end(st);
        return rc;
    }
    ReprojLoss p{};
    p.left = tensors["raw_left"].p; p.right = tensors["raw_right"].p;
    p.disp = disp[which].p; p.loss = scalars + slot;
    p.ddisp = with_grad ? g_disp.p : nullptr;
    p.workspace = ws; p.B = B; p.H = H; p.W = W; p.grad_scale = grad_scale;
    prof_begin(CAT_LOSS, st);
    int rc = reproj_loss(p, st);
    prof_end(st);
    return rc;
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
// every weight-gradient launch of the backward pass goes to `wstream`, ordered after the point of `st` that produced its
// operands; they share one workspace, so they serialise among themselves while the dgrad chain proceeds on `st`
int Engine::fork_wgrad(cudaStream_t st, cudaStream_t* ws) {
    *ws = st;
    if (profiling || net != 0) return 0;
    if (!wstream) {
        MS_CHECK_CUDA(cudaStreamCreateWithFlags(&wstream, cudaStreamNonBlocking));
        MS_CHECK_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
        MS_CHECK_CUDA(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
    }
    MS_CHECK_CUDA(cudaEventRecord(ev_fork, st));
    MS_CHECK_CUDA(cudaStreamWaitEvent(wstream, ev_fork, 0));
    wstream_dirty = true;
    *ws = wstream;
    return 0;
}
int Engine::join_wgrad(cudaStream_t st) {
    if (!wstream_dirty) return 0;
    wstream_dirty = false;
    MS_CHECK_CUDA(cudaEventRecord(ev_join, wstream));
    MS_CHECK_CUDA(cudaStreamWaitEvent(st, ev_join, 0));
    return 0;
}

int Engine::backward(int mode, int group, cudaStream_t st) {
    const int rc = backward_impl(mode, group, st);
    const int rj = join_wgrad(st);            // always: a captured side branch must be joined before the capture ends
    return rc ? rc : rj;
}

int Engine::backward_impl(int mode, int group, cudaStream_t st) {
    MS_REQUIRE(bound, "backward: engine not bound");
    if (net == 1) {
        // the reference cannot run MAD on DispNet either: 6 side predictions vs 5 groups trips the assert at
        // Stereo_Online_Adaptation.py:97
        MS_REQUIRE(mode == 2, "backward: DispNet supports FULL adaptation only");
        return backward_dispnet(st);
    }
    MS_REQUIRE(mode == 2 || (mode == 1 && group >= 0 && group < n_groups), "backward: bad mode/group");
    const int nd = (2 * radius_d) / corr_stride + 1;
    for (int i = 1; i <= 12; ++i) fresh.erase(g_pyr[i].p);     // gradient planes never survive from an earlier pass
    for (int k = 2; k <= 6; ++k) for (int j = 1; j <= 5; ++j) fresh.erase(g_est[k][j].p);
    for (int j = 1; j <= 6; ++j) fresh.erase(g_ctx[j].p);

    // lowest-index trainable pyramid conv (13 = none)
    int lo_pyr = 13;
    for (int i = 1; i <= 12; ++i) if (trainable(i - 1, mode, group)) { lo_pyr = i; break; }
    auto any_trainable = [&](int first, int last) {
        for (int i = first; i <= last; ++i) if (trainable(i, mode, group)) return true;
        return false;
    };

    // ---- estimator chain of level k: dpre(V_k) in g_V[k] -> (optionally) g_cost[k]
    auto est_bwd = [&](int k, bool need_cost_grad) -> int {
        for (int j = 6; j >= 1; --j) {
            const int li = est_layer(k, j);
            bool need_dx = (j > 1) ? (need_cost_grad || any_trainable(est_layer(k, 1), li - 1)) : need_cost_grad;
            if (conv_bwd(li, need_dx, j > 1 ? MAD_ALPHA : 1.f, 0, trainable(li, mode, group), st)) return -1;
            if (!need_dx) break;
        }
        return 0;
    };
    // ---- context chain: g_final -> g_ctxin
    auto ctx_bwd = [&](bool need_in_grad) -> int {
        for (int j = 7; j >= 1; --j) {
            const int li = ctx_layer(j);
            bool need_dx = (j > 1) ? (need_in_grad || any_trainable(ctx_layer(1), li - 1)) : need_in_grad;
            if (conv_bwd(li, need_dx, j > 1 ? MAD_ALPHA : 1.f, 0, trainable(li, mode, group), st)) return -1;
            if (!need_dx) break;
        }
        return 0;
    };
    // ---- correlation + warp backward of level k -> g_pyr[f] (left|right halves), optional g_u[k]
    auto corr_level_bwd = [&](int k, bool want_du) -> int {
        const int f = feat_of(k), C = PYR_CH[f];
        TView Lf = batch(pyr[f], 0, B), Rf = batch(pyr[f], B, B);
        TView dL = batch(g_pyr[f], 0, B), dR = batch(g_pyr[f], B, B);
        CorrBwd cb{};
        cb.left = Lf.p; cb.lcs = Lf.cs; cb.right = Rf.p; cb.rcs = Rf.cs;
        cb.u = (k < 6 && warping) ? slice(cost[k], C + nd, 1).p : nullptr; cb.ucs = cost[k].cs;
        cb.dcost = g_cost[k].p; cb.dcs = g_cost[k].cs;
        cb.dleft = dL.p; cb.dlcs = dL.cs; cb.dright = dR.p; cb.drcs = dR.cs;
        cb.du = (want_du && cb.u) ? g_u[k].p : nullptr; cb.ducs = 1;
        cb.B = B; cb.h = cost[k].h; cb.w = cost[k].w; cb.C = C; cb.max_disp = radius_d; cb.stride = corr_stride;
        cb.add_left_slice = 1; cb.acc_left = 0; cb.acc_right = 0; cb.gcoff = -1;
        fresh.erase(g_pyr[f].p);
        prof_begin(CAT_CORR_BWD, st);
        int crc = corr_bwd(cb, st);
        prof_end(st);
        prof_note(0, (double)B * cb.h * cb.w * (4.0 * C + nd) * 4.0);
        return crc;
    };
    // ---- pyramid: g_pyr[top] holds d(post-activation output of conv `top`), complete
    auto pyr_bwd = [&](int top, int lo, bool accumulate_feats) -> int {
        if (lo > top) return 0;
        fresh.erase(g_pyr[top].p);
        if (leaky_bwd(g_pyr[top].p, g_pyr[top].cs, pyr[top].p, pyr[top].cs, g_pyr[top].pixels(), g_pyr[top].c,
                      MAD_ALPHA, st)) return -1;
        for (int i = top; i >= lo; --i) {
            bool need_dx = i > lo;
            int acc = 0;
            if (need_dx && accumulate_feats && (i - 1) >= 4 && ((i - 1) % 2 == 0)) acc = 1;
            if (conv_bwd(i - 1, need_dx, MAD_ALPHA, acc, trainable(i - 1, mode, group), st)) return -1;
        }
        return 0;
    };
    auto ctx_tail = [&]() -> int {   // g_V[2] = g_final + g_ctxin[...,32]
        if (add_channels(g_V[2].p, 1, g_final.p, 1, g_final.pixels(), 1, 1.f, 0, st)) return -1;
        return add_channels(g_V[2].p, 1, g_ctxin.p + PYR_CH[4], g_ctxin.cs, g_final.pixels(), 1, 1.f, 1, st);
    };
    auto ctx_feat = [&]() -> int {   // g_pyr[4].left += g_ctxin[..., :32]
        TView dL = batch(g_pyr[4], 0, B);
        fresh.erase(g_pyr[4].p);
        return add_channels(dL.p, dL.cs, g_ctxin.p, g_ctxin.cs, dL.pixels(), PYR_CH[4], 1.f, 1, st);
    };

    if (mode == 1) {
        const int k = 6 - group;   // seed: disparity `group` of get_disparities() (D6,D5,D4,D3,D2ctx)
        MS_REQUIRE(k >= 2 && k <= 6, "backward(MAD): group has no disparity head");
        const int f = feat_of(k);
        const bool need_feat = lo_pyr <= f;
        const TView& head = (k == 2) ? final_ : V[k];
        TView& ghead = (k == 2) ? g_final : g_V[k];
        if (rs_scale > 1) {     // the module loss ran at 1/s resolution (loss): its gradient [B,h,w] is in g_disp
            const RsTables& t = rs_tab[group];
            if (rs_module_disp_bwd(g_disp.p, head.p, head.cs, B, head.h, head.w, t.rows, t.rrange, t.cols, t.crange, rs_disp.h,
                            rs_disp.w, ghead.p, 1, -20.f, rs_tmp, st)) return -1;
        } else if (resize_bilinear_bwd(g_disp.p, 1, head.p, head.cs, B, head.h, head.w, ghead.p, 1, Hp, Wp, H, W, -20.f, 1,
                                       1.f, 0, 0, rs_tmp, st)) return -1;
        if (k == 2) {
            bool est_train = any_trainable(est_layer(2, 1), est_layer(2, 6));
            if (ctx_bwd(need_feat || est_train)) return -1;
            if (need_feat || est_train) { if (ctx_tail()) return -1; }
            else return 0;
        }
        if (est_bwd(k, need_feat)) return -1;
        if (!need_feat) return 0;
        if (corr_level_bwd(k, false)) return -1;
        if (k == 2 && ctx_feat()) return -1;
        return pyr_bwd(f, lo_pyr, false);
    }

    // ---- FULL: loss on disp[5] = relu(resize(final)*-20)
    if (resize_bilinear_bwd(g_disp.p, 1, final_.p, final_.cs, B, final_.h, final_.w, g_final.p, 1, Hp, Wp, H, W, 1.f, 0,
                            -20.f, 1, 0, rs_tmp, st)) return -1;
    if (ctx_bwd(true)) return -1;
    if (ctx_tail()) return -1;
    for (int k = 2; k <= 6; ++k) {
        const int f = feat_of(k), C = PYR_CH[f];
        if (est_bwd(k, true)) return -1;
        if (corr_level_bwd(k, true)) return -1;
        if (k == 2 && ctx_feat()) return -1;
        if (k < 6) {
            // d u_k = warp-coordinate grad (if warping) + estimator-input slice
            const int acc = warping ? 1 : 0;
            if (add_channels(g_u[k].p, 1, g_cost[k].p + C + nd, g_cost[k].cs, g_u[k].pixels(), 1, 1.f, acc, st)) return -1;
            if (resize_bilinear_bwd(g_u[k].p, 1, V[k + 1].p, V[k + 1].cs, B, V[k + 1].h, V[k + 1].w, g_V[k + 1].p, 1,
                                    cost[k].h, cost[k].w, cost[k].h, cost[k].w, 1.f, 0, 20.f / (float)(1 << k), 0, 0,
                                    rs_tmp, st)) return -1;
        }
    }
    return pyr_bwd(12, 1, true);
}

int Engine::update(int group, float lr, float mu, float gscale, cudaStream_t st) {
    MS_REQUIRE(bound, "engine not bound");
    size_t b = 0, e = n_params;
    if (group >= 0) { MS_REQUIRE(group < n_groups, "update: bad group"); b = group_begin[group]; e = group_end[group]; }
    if (opt_kind == 1) {
        if (adam_update(Wt + b, Gr + b, Mo + b, adam_v + b, adam_powers, e - b, lr, adam_b1, adam_b2, adam_eps, gscale, st))
            return -1;
    } else if (momentum_update(Wt + b, Gr + b, Mo + b, e - b, lr, mu, gscale, st)) {
        return -1;
    }
    return prep_layers(group, st);      // refresh the 16-bit weight tiles of exactly the weights that moved
}

// Only while a step graph is captured without instrumentation (run() calls run_eager directly only to profile), and only
// when no layer of the module runs after its disparity head: its update must not move weights the forward's tail reads.
bool Engine::mad_branch(int mode, int group) const {
    if (mode != 1 || profiling || net != 0 || group < 0 || group > 4) return false;
    const int head = group < 4 ? est_layer(6 - group, 6) : ctx_layer(7);     // layers are indexed in forward order
    for (size_t li = 0; li < layers.size(); ++li)
        if (layers[li].group == group && (int)li > head) return false;
    return true;
}

// forward + losses + backward (+ update) as one sequence; replayed as a CUDA graph after the first call
int Engine::run_eager(int mode, int group, int disp_mask, int with_update, float lr, float mu, float gscale,
                      cudaStream_t st) {
    const int full = n_disp - 1;
    int mask = disp_mask | (1 << full);
    const bool rs = mode == 1 && rs_scale > 1 && net == 0;     // module loss at 1/s: read straight from the coarse head
    if (mode == 1 && !rs) mask |= 1 << group;
    // NVTX ranges (SURVEY section 5: tracing): visible in nsys / ncu timelines, free when no tool is attached
    struct Range { explicit Range(const char* n) { nvtxRangePushA(n); } ~Range() { nvtxRangePop(); } };
    const bool branch = mad_branch(mode, group);
    if (branch && !bstream) {
        MS_CHECK_CUDA(cudaStreamCreateWithFlags(&bstream, cudaStreamNonBlocking));
        MS_CHECK_CUDA(cudaEventCreateWithFlags(&ev_bfork, cudaEventDisableTiming));
        MS_CHECK_CUDA(cudaEventCreateWithFlags(&ev_bjoin, cudaEventDisableTiming));
    }
    cudaStream_t bs = branch ? bstream : st;     // the train op's stream
    if (rs) {       // the loss-resolution images only need the input: on the train op's stream, beside the forward
        Range r("madstereo/loss_inputs");
        if (branch) {
            MS_CHECK_CUDA(cudaEventRecord(ev_bfork, st));
            MS_CHECK_CUDA(cudaStreamWaitEvent(bs, ev_bfork, 0));
        }
        const bool pdl = pdl_enabled();
        if (branch) pdl_set_suppressed(true);
        const int rc = rs_prepare_inputs(bs);
        pdl_set_suppressed(!pdl);
        if (rc) return rc;
    }
    { Range r("madstereo/forward"); if (forward(mask, st, branch ? group : -1, branch ? bstream : nullptr)) return -1; }
    { Range r("madstereo/loss_full"); if (loss(full, mode == 2, 0, 1.f, st)) return -1; }
    if (mode == 1) {
        auto train_op = [&]() -> int {
            { Range r("madstereo/loss_module"); if (loss(group, 1, 1, 1.f, bs)) return -1; }
            { Range r("madstereo/backward_mad"); if (backward(1, group, bs)) return -1; }
            Range r("madstereo/update");
            return with_update == 1 ? update(group, lr, mu, gscale, bs) : 0;
        };
        // The branch's kernels launch without PDL: their CTAs would otherwise become resident early and wait in
        // griddepcontrol.wait, holding SM resources that the forward's tail and the weight gradients beside them could
        // use (tools/step_phases.py: faster for every module, most for module 4, whose dgrad chain is the longest)
        const bool pdl = pdl_enabled();
        on_branch = branch ? 1 : 0;
        if (branch) pdl_set_suppressed(true);
        const int rc = train_op();
        pdl_set_suppressed(!pdl);
        on_branch = 0;
        if (branch) {       // always joined: a captured side branch must be joined before the capture ends
            MS_CHECK_CUDA(cudaEventRecord(ev_bjoin, bs));
            MS_CHECK_CUDA(cudaStreamWaitEvent(st, ev_bjoin, 0));
        }
        if (rc) return rc;
        // all-reduce over peer memory + update: reads both loss slots and waits for the peers, so never beside the forward
        if (with_update == 2 && dp_update(group, lr, mu, st)) return -1;
    } else if (mode == 2) {
        { Range r("madstereo/backward_full"); if (backward(2, 0, st)) return -1; }
        Range r("madstereo/update");
        if (with_update == 1 && update(-1, lr, mu, gscale, st)) return -1;
        if (with_update == 2 && dp_update(-1, lr, mu, st)) return -1;
    }
    return 0;
}

int Engine::run(int mode, int group, int disp_mask, int with_update, float lr, float mu, float gscale, cudaStream_t st) {
    MS_REQUIRE(bound, "engine not bound");
    MS_REQUIRE(mode == 0 || mode == 2 || (mode == 1 && group >= 0 && group < n_groups), "run: bad mode/group");
    MS_REQUIRE(!(with_update == 2 && mode != 0 && opt_kind != 0),
               "run: the fused data-parallel exchange (with_update=2) applies momentum only; Adam is single-GPU");
    if (profiling == 1) return run_eager(mode, group, disp_mask, with_update, lr, mu, gscale, st);
    if (weights_dirty) {                    // load / restore happened: refresh every weight tile outside the graph
        if (prep_layers(-1, st)) return -1;
        weights_dirty = false;
    }
    if (!gstream) {
        MS_CHECK_CUDA(cudaStreamCreateWithFlags(&gstream, cudaStreamNonBlocking));
        MS_CHECK_CUDA(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
        MS_CHECK_CUDA(cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming));
    }
    GraphKey key;
    memset(&key, 0, sizeof key);
    key.mode = mode; key.group = mode == 1 ? group : 0; key.mask = disp_mask; key.with_update = with_update;
    key.lr = lr; key.mu = mu; key.gs = gscale; key.prof = profiling == 2 ? 1 : 0;
    auto it = graphs.find(key);
    if (it == graphs.end()) {
        if (conv_bf_init() || wgrad_bf_init() || corr_init()) return -1;
        cudaGraph_t graph = nullptr;
        const long long l0 = launch_count();
        if (profiling == 2) { if (prof_collect()) return -1; }
        MS_CHECK_CUDA(cudaStreamBeginCapture(gstream, cudaStreamCaptureModeThreadLocal));
        prof_capturing = profiling == 2;
        pdl_set_suppressed(prof_capturing);
        if (prof_capturing) { prof_begin(-1, gstream); prof_end(gstream); }      // calibration span (see prof_fold)
        int rc = run_eager(mode, group, disp_mask, with_update, lr, mu, gscale, gstream);
        prof_capturing = false;
        pdl_set_suppressed(false);
        cudaError_t ce = cudaStreamEndCapture(gstream, &graph);
        if (rc) { if (graph) cudaGraphDestroy(graph); spans.clear(); return rc; }
        MS_CHECK_CUDA(ce);
        cudaGraphExec_t exec = nullptr;
        MS_CHECK_CUDA(cudaGraphInstantiate(&exec, graph, 0));
        cudaGraphDestroy(graph);
        GraphRec rec{exec, launch_count() - l0, nullptr};
        if (profiling == 2) { rec.spans = new std::vector<Span>(spans); spans.clear(); }
        add_launches(-rec.kernels);            // counted again at every replay below
        it = graphs.emplace(key, rec).first;
    }
    // order: caller's stream -> private stream (graph) -> caller's stream
    MS_CHECK_CUDA(cudaEventRecord(ev_in, st));
    MS_CHECK_CUDA(cudaStreamWaitEvent(gstream, ev_in, 0));
    MS_CHECK_CUDA(cudaGraphLaunch(it->second.exec, gstream));
    add_launches(it->second.kernels);
    if (mode == 1 && rs_scale > 1) rs_fresh = true;     // the step wrote this frame's loss-resolution inputs
    MS_CHECK_CUDA(cudaEventRecord(ev_out, gstream));
    MS_CHECK_CUDA(cudaStreamWaitEvent(st, ev_out, 0));
    if (profiling == 2 && it->second.spans) {        // in-graph timing: read the event nodes of THIS replay
        MS_CHECK_CUDA(cudaStreamSynchronize(gstream));
        if (prof_fold(*it->second.spans, false)) return -1;
    }
    return 0;
}

}  // namespace ms
