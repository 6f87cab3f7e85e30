// DispNet-C schedule for the engine: forward and FULL backward (see engine.h).
//
// Graph restated from the reference (never copied): Nets/DispNet.py:75-152 (_build_network, correlation=True),
// :45-57 (_upsampling_block: deconv 4x4 s2, predict 3x3 -> 1, up_predict 4x4 s2 1 -> 1, concat 3x3 linear),
// :39-43 (_make_disp), :59-73 (input normalisation), MAX_DISP=40 (:7).  conv2d default activation = leaky 0.1
// (Nets/sharedLayers.py:54).  MAD is not defined for DispNet in the reference (assert at
// Stereo_Online_Adaptation.py:97), so only NONE / FULL exist here.
#include <algorithm>

#include "engine.h"

namespace ms {

static const float DN_ALPHA = 0.1f;
static const int DN_MAXD = 40;
struct EncSpec { const char* scope; const char* name; int k, cin, cout, stride; };
static const EncSpec DN_ENC[11] = {
    {"conv1", "conv1a", 7, 3, 64, 2},        {"conv2", "conv2a", 5, 64, 128, 2},     {"conv_redir", "conv_redir", 1, 128, 64, 1},
    {"conv3", "conv3", 5, 145, 256, 2},      {"conv3/1", "conv3/1", 3, 256, 256, 1}, {"conv4", "conv4", 3, 256, 512, 2},
    {"conv4/1", "conv4/1", 3, 512, 512, 1},  {"conv5", "conv5", 3, 512, 512, 2},     {"conv5/1", "conv5/1", 3, 512, 512, 1},
    {"conv6", "conv6", 3, 512, 1024, 2},     {"conv6/1", "conv6/1", 3, 1024, 1024, 1}};
struct UpSpec { const char* name; int cin, cout, skip; };
static const UpSpec DN_UP[5] = {{"up5", 1024, 512, 512}, {"up4", 512, 256, 512}, {"up3", 256, 128, 256},
                                {"up2", 128, 64, 128},   {"up1", 64, 32, 64}};
static inline int up_layer(int u, int j) { return 11 + 4 * u + j; }   // j: 0 deconv, 1 predict, 2 up_predict, 3 concat
static const int DN_PRED = 31;
static inline int pad4i(int c) { return (c + 3) / 4 * 4; }

int Engine::build_dispnet() {
    layers.clear();
    auto add = [&](const std::string& name, const std::string& scope, int k, int cin, int cout, int stride, float alpha,
                   int transposed) {
        ConvLayer L;
        L.name = name; L.scope = "model/" + scope; L.bname = "bias";
        L.kh = L.kw = k; L.cin = cin; L.cout = cout; L.stride = stride; L.dil = 1; L.alpha = alpha;
        L.transposed = transposed; L.group = -1; L.w_off = L.b_off = 0;
        layers.push_back(L);
    };
    for (const auto& e : DN_ENC) add(e.name, e.scope, e.k, e.cin, e.cout, e.stride, DN_ALPHA, 0);
    for (const auto& u : DN_UP) {
        std::string n(u.name);
        add(n + "/deconv", n + "/deconv", 4, u.cin, u.cout, 2, DN_ALPHA, 1);
        add(n + "/predict", n + "/predict", 3, u.cin, 1, 1, 1.f, 0);
        add(n + "/up_predict", n + "/up_predict", 4, 1, 1, 2, 1.f, 1);
        add(n + "/concat", n + "/concat", 3, u.cout + u.skip + 1, u.cout, 1, 1.f, 0);
    }
    add("prediction", "prediction", 3, 32, 1, 1, 1.f, 0);
    radius_d = DN_MAXD; corr_stride = 1; warping = 0;
    return 0;
}

void Engine::layout_dispnet(Bump& A) {
    const int h2 = Hp / 2, w2 = Wp / 2, h4 = Hp / 4, w4 = Wp / 4, nd = 2 * DN_MAXD + 1;
    d_c1 = A.tens(2 * B, h2, w2, 64); gd_c1 = A.tens(2 * B, h2, w2, 64);
    d_c2 = A.tens(2 * B, h4, w4, 128); gd_c2 = A.tens(2 * B, h4, w4, 128);
    d_cat3 = A.tens(B, h4, w4, 145, 148); gd_cat3 = A.tens(B, h4, w4, 145, 148);
    plan_views(0, img, d_c1, gd_c1, TView{});
    plan_views(1, d_c1, d_c2, gd_c2, gd_c1);
    plan_views(2, batch(d_c2, 0, B), slice(d_cat3, nd, 64), slice(gd_cat3, nd, 64), batch(gd_c2, 0, B));
    int hh = h4, ww = w4;
    for (int i = 0; i < 8; ++i) {
        const ConvLayer& L = layers[3 + i];
        if (L.stride == 2) { hh /= 2; ww /= 2; }
        d_enc[i] = A.tens(B, hh, ww, L.cout); gd_enc[i] = A.tens(B, hh, ww, L.cout);
        plan_views(3 + i, i ? d_enc[i - 1] : d_cat3, d_enc[i], gd_enc[i], i ? gd_enc[i - 1] : gd_cat3);
        tensors[L.name] = d_enc[i]; tensors["grad/" + L.name] = gd_enc[i];
    }
    tensors["conv1a"] = batch(d_c1, 0, B); tensors["conv1b"] = batch(d_c1, B, B);
    tensors["conv2a"] = batch(d_c2, 0, B); tensors["conv2b"] = batch(d_c2, B, B);
    tensors["corr"] = slice(d_cat3, 0, nd);
    tensors["conv_redir"] = slice(d_cat3, nd, 64);
    tensors["grad/conv1"] = gd_c1; tensors["grad/conv2"] = gd_c2; tensors["grad/cat3"] = gd_cat3;
    // decoder: bottom of up5 is conv6/1 at Hp/64
    int bh = Hp / 64, bw = Wp / 64;
    for (int u = 0; u < 5; ++u) {
        const UpSpec& S = DN_UP[u];
        const int ct = S.skip + S.cout + 1;
        d_pr[u] = A.tens(B, bh, bw, 1); gd_pr[u] = A.tens(B, bh, bw, 1);
        d_cat[u] = A.tens(B, 2 * bh, 2 * bw, ct, pad4i(ct)); gd_cat[u] = A.tens(B, 2 * bh, 2 * bw, ct, pad4i(ct));
        d_cc[u] = A.tens(B, 2 * bh, 2 * bw, S.cout); gd_cc[u] = A.tens(B, 2 * bh, 2 * bw, S.cout);
        const TView bottom = u ? d_cc[u - 1] : d_enc[7], gbottom = u ? gd_cc[u - 1] : gd_enc[7];
        // (the deconv output's gradient is a channel slice of gd_cat[u]: its planes are compact, keyed by the slice)
        plan_views(up_layer(u, 0), bottom, slice(d_cat[u], S.skip, S.cout), slice(gd_cat[u], S.skip, S.cout), gbottom);
        plan_views(up_layer(u, 1), bottom, d_pr[u], gd_pr[u], gbottom);
        plan_views(up_layer(u, 2), d_pr[u], slice(d_cat[u], S.skip + S.cout, 1), slice(gd_cat[u], S.skip + S.cout, 1), gd_pr[u]);
        plan_views(up_layer(u, 3), d_cat[u], d_cc[u], gd_cc[u], gd_cat[u]);
        std::string n(S.name);
        tensors[n + "/predict"] = d_pr[u];
        tensors[n + "/deconv"] = slice(d_cat[u], S.skip, S.cout);
        tensors[n + "/up_predict"] = slice(d_cat[u], S.skip + S.cout, 1);
        tensors[n + "/concat"] = d_cc[u];
        tensors["grad/" + n + "/concat"] = gd_cc[u];
        tensors[n + "/cat"] = d_cat[u]; tensors["grad/" + n + "/cat"] = gd_cat[u];    // [skip | deconv | up_predict]
        tensors["grad/" + n + "/predict"] = gd_pr[u];
        bh *= 2; bw *= 2;
    }
    d_pred = A.tens(B, h2, w2, 1); gd_pred = A.tens(B, h2, w2, 1);
    plan_views(DN_PRED, d_cc[4], d_pred, gd_pred, gd_cc[4]);
    tensors["prediction"] = d_pred; tensors["grad/prediction"] = gd_pred;
}

int Engine::forward_dispnet(int disp_mask, cudaStream_t st) {
    const int nd = 2 * DN_MAXD + 1;
    for (int li = 0; li < 3; ++li)          // conv1, conv2, conv_redir
        if (conv_fwd(li, nullptr, 0, st)) return -1;
    TView c2a = batch(d_c2, 0, B), c2b = batch(d_c2, B, B);
    {
        CorrFwd cf{};
        cf.left = c2a.p; cf.lcs = c2a.cs; cf.right = c2b.p; cf.rcs = c2b.cs; cf.u = nullptr; cf.ucs = 0;
        cf.out = d_cat3.p; cf.ocs = d_cat3.cs; cf.out2 = nullptr; cf.o2cs = 0;
        cf.B = B; cf.h = d_c2.h; cf.w = d_c2.w; cf.C = 128; cf.max_disp = DN_MAXD; cf.stride = 1; cf.copy_left = 0; cf.u_chan = 0;
        cf.plane_scale = act_scale;   // same fp16 hi/lo arithmetic as the forward convs
        prof_begin(CAT_CORR_FWD, st);
        int rc = corr_fwd(cf, st);
        prof_end(st);
        prof_note(0, (double)B * cf.h * cf.w * (2.0 * 128 + nd) * 4.0);
        if (rc) return -1;
    }
    for (int i = 0; i < 8; ++i)
        if (conv_fwd(3 + i, nullptr, 0, st)) return -1;
    const TView skips[5] = {d_enc[5], d_enc[3], d_enc[1], c2a, batch(d_c1, 0, B)};
    for (int u = 0; u < 5; ++u) {
        const TView& cat = d_cat[u];
        if (add_channels(cat.p, cat.cs, skips[u].p, skips[u].cs, cat.pixels(), DN_UP[u].skip, 1.f, 0, st)) return -1;   // tf.concat copy
        for (int j = 0; j < 4; ++j)         // deconv, predict, up_predict, concat
            if (conv_fwd(up_layer(u, j), nullptr, 0, st)) return -1;
    }
    if (conv_fwd(DN_PRED, nullptr, 0, st)) return -1;
    for (int i = 0; i < 7; ++i) {
        if (!(disp_mask & (1 << i))) continue;
        const TView& src = i < 5 ? d_pr[i] : d_pred;
        if (i < 6) {   // _make_disp: resize(relu(op * Wp/w_op))
            if (resize_bilinear(src.p, src.cs, B, src.h, src.w, disp[i].p, 1, Hp, Wp, H, W, (float)Wp / (float)src.w, 1, 1.f, 0, st)) return -1;
        } else {       // rescaled_prediction = resize(prediction) * 2, no relu (DispNet.py:149)
            if (resize_bilinear(src.p, src.cs, B, src.h, src.w, disp[i].p, 1, Hp, Wp, H, W, 1.f, 0, 2.f, 0, st)) return -1;
        }
    }
    return 0;
}

// conv2d_transpose backward of layer li, always with its weight gradient and with the input gradient into its planned dx
// (dx_acc: added to it).  x: its input [n,h,w,cin]; dpre: grad wrt pre-activation output [n,2h,2w,cout].
//   dW[kh,kw,cout,cin] = wgrad of the stride-2 conv that maps the big map (channels cout) to the small one (channels cin)
//   dx                 = that stride-2 conv applied to dpre with the same (canonical) weights as HWIO [.,.,cout,cin]
int Engine::deconv_bwd(int li, int dx_acc, cudaStream_t st) {
    const ConvLayer& L = layers[li];
    const ConvPlan& P = plan[li];
    MS_REQUIRE(L.transposed, "deconv_bwd: not a transposed layer");
    MS_REQUIRE(P.dx.p, "deconv_bwd: layer " + L.name + " has no planned input gradient");
    ConvWgrad q;
    ConvGemm p;
    wgrad_args(li, q);                      // (both fit: plan_convs checked the plan's views)
    dgrad_args(li, p);
    if (P.dp) { fresh.erase(P.dpre.p); if (ensure_planes(P.dpre, P.dp, st)) return -1; }     // bf16 planes of the big map's gradient
    {
        prof_begin(CAT_CONV_WGRAD, st, li);
        int rc = wgrad(L, P, q, st);
        if (!rc) rc = bias_grad(P.dpre, Gr + L.b_off, wg_ws, wg_ws_floats, st);
        prof_end(st);
        prof_note((double)P.x.pixels() * L.kh * L.kw * L.cin * L.cout, 0);
        if (rc) return -1;
    }
    p.accumulate = dx_acc;
    prof_begin(CAT_CONV_DGRAD, st, li);
    // (an accumulating launch would leave dx's own planes stale: it writes none)
    const int rc = P.dgrad == ConvPlan::DGRAD_BF ? conv_bf(p, *P.dp, P.tiles[1], nullptr, sk().bf_part, sk().bf_tickets, st) : conv_gemm(p, st);
    planes_written(P.dx, P.dxp, false);
    prof_end(st);
    prof_note((double)P.x.pixels() * L.kh * L.kw * L.cin * L.cout, 0);
    return rc ? -1 : 0;
}

int Engine::backward_dispnet(cudaStream_t st) {
    const int nd = 2 * DN_MAXD + 1;
    // loss on disp[6] = crop(resize(prediction) * 2)
    if (resize_bilinear_bwd(g_disp.p, 1, d_pred.p, d_pred.cs, B, d_pred.h, d_pred.w, gd_pred.p, 1, Hp, Wp, H, W, 1.f, 0, 2.f, 0,
                            0, rs_tmp, st)) return -1;
    // prediction conv (linear): -> grad of up1/concat output
    if (conv_bwd(DN_PRED, 1, 1.f, 0, 1, st)) return -1;

    for (int u = 4; u >= 0; --u) {
        const UpSpec& S = DN_UP[u];
        // concat conv (linear): dpre = gd_cc[u] ; input = d_cat[u]
        if (conv_bwd(up_layer(u, 3), 1, 1.f, 0, 1, st)) return -1;
        TView g_dec = slice(gd_cat[u], S.skip, S.cout), dec_act = slice(d_cat[u], S.skip, S.cout);
        if (leaky_bwd(g_dec.p, g_dec.cs, dec_act.p, dec_act.cs, g_dec.pixels(), S.cout, DN_ALPHA, st)) return -1;
        // up_predict (transposed, linear): input = predict output
        if (deconv_bwd(up_layer(u, 2), 0, st)) return -1;
        // predict conv (linear): dpre = gd_pr[u] -> grad of the bottom (write)
        if (conv_bwd(up_layer(u, 1), 1, 1.f, 0, 1, st)) return -1;
        // deconv (transposed, leaky already applied): -> grad of the bottom (accumulate)
        if (deconv_bwd(up_layer(u, 0), 1, st)) return -1;
    }
    // ---- encoder, top down.  gd_enc[7] = d(conv6/1 output) complete.
    // feature grads that also receive a skip-slice contribution: enc[5] (up5), enc[3] (up4), enc[1] (up3)
    auto skip_slice = [&](int u) { return slice(gd_cat[u], 0, DN_UP[u].skip); };
    if (leaky_bwd(gd_enc[7].p, gd_enc[7].cs, d_enc[7].p, d_enc[7].cs, gd_enc[7].pixels(), gd_enc[7].c, DN_ALPHA, st)) return -1;
    for (int i = 7; i >= 0; --i) {
        const TView& dx = i == 0 ? gd_cat3 : gd_enc[i - 1];
        int acc = 0;
        const int below = i - 1;              // index of the feature receiving dx
        int skip_u = below == 5 ? 0 : (below == 3 ? 1 : (below == 1 ? 2 : -1));
        if (skip_u >= 0) {                    // seed with the skip-connection gradient, then accumulate the dgrad
            TView sl = skip_slice(skip_u);
            if (add_channels(dx.p, dx.cs, sl.p, sl.cs, dx.pixels(), dx.c, 1.f, 0, st)) return -1;
            acc = 1;
        }
        if (conv_bwd(3 + i, 1, i == 0 ? 1.f : DN_ALPHA, acc, 1, st)) return -1;
    }
    // gd_cat3: [0,81) corr grads (linear), [81,145) conv_redir output grads (leaky)
    {
        TView g_red = slice(gd_cat3, nd, 64), red_act = slice(d_cat3, nd, 64);
        if (leaky_bwd(g_red.p, g_red.cs, red_act.p, red_act.cs, g_red.pixels(), 64, DN_ALPHA, st)) return -1;
        TView gc2a = batch(gd_c2, 0, B), gc2b = batch(gd_c2, B, B);
        if (conv_bwd(2, 1, 1.f, 0, 1, st)) return -1;           // conv_redir: writes d(conv2a)
        CorrBwd cb{};
        TView c2a = batch(d_c2, 0, B), c2b = batch(d_c2, B, B);
        cb.left = c2a.p; cb.lcs = c2a.cs; cb.right = c2b.p; cb.rcs = c2b.cs; cb.u = nullptr; cb.ucs = 0;
        cb.dcost = gd_cat3.p; cb.dcs = gd_cat3.cs; cb.dleft = gc2a.p; cb.dlcs = gc2a.cs; cb.dright = gc2b.p; cb.drcs = gc2b.cs;
        cb.du = nullptr; cb.ducs = 0;
        cb.B = B; cb.h = d_c2.h; cb.w = d_c2.w; cb.C = 128; cb.max_disp = DN_MAXD; cb.stride = 1;
        cb.add_left_slice = 0; cb.acc_left = 1; cb.acc_right = 0; cb.gcoff = 0;
        prof_begin(CAT_CORR_BWD, st);
        int rc = corr_bwd(cb, st);
        prof_end(st);
        prof_note(0, (double)B * cb.h * cb.w * (4.0 * 128 + nd) * 4.0);
        if (rc) return -1;
        TView sl = skip_slice(3);                                                                   // up2 skip = conv2a
        if (add_channels(gc2a.p, gc2a.cs, sl.p, sl.cs, gc2a.pixels(), 128, 1.f, 1, st)) return -1;
    }
    if (leaky_bwd(gd_c2.p, gd_c2.cs, d_c2.p, d_c2.cs, gd_c2.pixels(), 128, DN_ALPHA, st)) return -1;
    // conv2 (shared, batch 2B): wgrad + dgrad -> gd_c1 ; then the up1 skip (conv1a) ; then leaky
    if (conv_bwd(1, 1, 1.f, 0, 1, st)) return -1;
    {
        TView gc1a = batch(gd_c1, 0, B), sl = skip_slice(4);
        if (add_channels(gc1a.p, gc1a.cs, sl.p, sl.cs, gc1a.pixels(), 64, 1.f, 1, st)) return -1;
    }
    if (leaky_bwd(gd_c1.p, gd_c1.cs, d_c1.p, d_c1.cs, gd_c1.pixels(), 64, DN_ALPHA, st)) return -1;
    return conv_bwd(0, 0, 1.f, 0, 1, st);
}

}  // namespace ms
