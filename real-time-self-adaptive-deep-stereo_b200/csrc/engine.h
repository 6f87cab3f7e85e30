// Engine: per-frame MADNet / DispNet forward + (MAD | FULL) backward + momentum update, orchestrated in C++
// over caller-owned device memory.  Replaces what one `sess.run(fetches)` executes in the reference's inner
// loop (Stereo_Online_Adaptation.py:208) for the graphs built by Nets/MadNet.py and Nets/DispNet.py.
#pragma once
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "common.cuh"

namespace ms {

struct ConvLayer {
    std::string name;     // reference layer name as used in block_config JSON ("left/conv1", "context3", ...)
    std::string scope;    // TF variable scope ("model/gc-read-pyramid/conv1")
    std::string bname;    // "biases" (MADNet) or "bias" (DispNet)
    int kh, kw, cin, cout, stride, dil;
    float alpha;          // leaky slope, 1 = linear
    int transposed;       // conv2d_transpose (weights [kh,kw,cout,cin])
    size_t w_off, b_off;  // float offsets in the parameter arena
    int group;            // MAD module index or -1
};

// The gather-GEMM encoding of a layer's three directions on the given views: SAME padding, the mul / off / step / div of
// the gather (a transposed layer's forward: the fractionally strided case) and the swapped operands of a transposed
// layer's weight gradient.  Fills the geometry fields and alpha and no pointer but the views'; false: the views do not
// fit the layer.  The engine and the per-op entry points (capi.cu) build every convolution from these.
bool conv_fwd_geom(const ConvLayer& L, const TView& x, const TView& y, ConvGemm& p);
bool conv_dgrad_geom(const ConvLayer& L, const TView& dpre, const TView& dx, ConvGemm& p);
bool conv_wgrad_geom(const ConvLayer& L, const TView& x, const TView& dpre, ConvWgrad& q);
// rows (columns) of the layer's output on `in` input rows (columns)
inline int conv_out_size(const ConvLayer& L, int in) { return L.transposed ? in * L.stride : (in + L.stride - 1) / L.stride; }

constexpr int DP_MAX_WORLD = 8;
struct DpState {               // device-resident exchange state of one rank (IPC-mapped into every peer), csrc/dp.cu
    unsigned int ready[DP_MAX_WORLD];   // ready[src] = (epoch << 8) | module tag, written by rank src
    unsigned int done[DP_MAX_WORLD];    // done[src]  = last epoch rank src finished reading this rank's buffer
    unsigned int epoch, blocks_done, error, pad;
};

// Which kernel runs each direction of a layer.  Engine::plan_convs() decides it once per layout from the views the
// layer runs on, with the kernels' own *_supported / conv_head_kind predicates, and allocates exactly what the chosen
// kernels read; conv_fwd / conv_bwd / deconv_bwd only switch on it.
struct ConvPlan {
    enum Fwd { FWD_HEAD, FWD_ONE_CHANNEL, FWD_STEM, FWD_SMALL, FWD_BF, FWD_GEMM } fwd;
    enum Dgrad { DGRAD_HEAD, DGRAD_BF, DGRAD_GEMM } dgrad;
    enum Wgrad { WGRAD_BF, WGRAD_STEM, WGRAD_HEAD, WGRAD_FP32 } wgrad;   // FP32: conv_wgrad, which picks its own kernel
    TView x, y, dpre, dx;                  // forward input / output, output and input gradients (dx.p == nullptr: none)
    void* tiles[2];                        // split 16-bit weight tiles of a BF forward (0) and a BF dgrad (1)
    const ActPlanes *xp, *yp, *dp, *dxp;   // 16-bit planes of x, y, dpre, dx; nullptr where no chosen kernel reads them
};

struct Bump {            // workspace bump allocator
    float* base; size_t off;
    float* alloc(size_t n) { float* p = base + off; off += (n + 63) / 64 * 64; return p; }
    TView tens(int n, int h, int w, int c, int cs = 0) { cs = cs ? cs : c; return view(alloc((size_t)n * h * w * cs), n, h, w, c, cs); }
};

// byte offset of the right frame in the uint8 staging buffer: the left frame's n bytes rounded up to 4
inline size_t u8_stage_right_offset(size_t n) { return (n + 3) & ~(size_t)3; }

struct Engine {
    // configuration
    int net;              // 0 = MADNet, 1 = DispNet
    int B, H, W, Hp, Wp;
    int radius_d, corr_stride, warping;
    std::vector<ConvLayer> layers;
    int n_groups;
    std::vector<size_t> group_begin, group_end;   // float ranges in the arena
    size_t n_params;      // arena floats (incl. alignment pads)

    // bound memory
    float *Wt, *Gr, *Mo;  // weights / grads / momentum arenas
    float* ws; size_t ws_floats;
    bool bound;

    // tensors (valid after bind)
    std::map<std::string, TView> tensors;

    // ---- MADNet buffers
    TView img;                       // [2B,Hp,Wp,3] cs=4
    TView pyr[13], g_pyr[13];        // 1..12
    TView cost[7], g_cost[7];        // levels 2..6
    TView est[7][7], g_est[7][7];    // [level][1..5]
    TView V[7], g_V[7];              // [level] (V[2] is a slice of ctxin)
    TView g_u[7];
    TView ctxin, g_ctxin, ctx[8], g_ctx[8], final_, g_final;
    TView disp[7];                   // MADNet: D6,D5,D4,D3,D2ctx,full ; DispNet: up5..up1 predict, prediction, full
    int n_disp;
    TView g_disp;
    float* wT; size_t wT_floats;     // transposed-weight scratch
    // split-K scratch: partial sums of conv_bf (with its self-resetting tickets) and of the CUDA-core conv (conv_gemm) on
    // small maps.  Set 0 serves the forward and every serial pass; set 1 the MAD train op that runs beside the rest of the
    // forward (mad_branch) -- it aliases set 0 where no such branch can run, and set 0's conv_gemm partials where no MAD
    // module's dgrad runs on conv_gemm.  Both sets have the same sizes, so the kernels split K the same way on either.
    struct SplitK { float* bf_part; unsigned int* bf_tickets; float* gemm_part; };
    SplitK splitk[2];
    int on_branch;                   // which set the launches being enqueued use
    const SplitK& sk() const { return splitk[on_branch]; }
    bool weights_dirty;
    // refreshes the tensor-core weight tiles of a module's layers right after its momentum update (-1 = all, after load/restore)
    int prep_layers(int group, cudaStream_t st);
    // whole-step CUDA graphs keyed by (mode, group, disp_mask, with_update, lr, mu, gscale)
    struct GraphKey { int mode, group, mask, with_update, prof; float lr, mu, gs;
                      bool operator<(const GraphKey& o) const { return memcmp(this, &o, sizeof(GraphKey)) < 0; } };
    struct Span;
    struct GraphRec { cudaGraphExec_t exec; long long kernels; std::vector<Span>* spans; };
    std::map<GraphKey, GraphRec> graphs;
    cudaStream_t gstream; cudaEvent_t ev_in, ev_out;   // graphs run on a private stream (the legacy default stream cannot be captured)
    // weight gradients on a side stream: wgrad(layer j) only needs dpre_j and the forward activation, so it runs concurrently
    // with the dgrad chain (fork / join through events; inside the captured step this becomes a parallel graph branch).
    // MADNet only, and off while profiling
    cudaStream_t wstream; cudaEvent_t ev_fork, ev_join; bool wstream_dirty;
    int fork_wgrad(cudaStream_t st, cudaStream_t* ws);
    int join_wgrad(cudaStream_t st);
    // MAD train op on a branch of the captured step: module g's loss, backward and update read only forward tensors that
    // exist once its disparity head has run (level 6-g's disp6, or context7 for the last module) and that nothing later in
    // the forward writes, so they run on `bstream` beside the rest of the forward.  MADNet only, and off while profiling
    bool mad_branch(int mode, int group) const;
    cudaStream_t bstream; cudaEvent_t ev_bfork, ev_bjoin;
    int backward_impl(int mode, int group, cudaStream_t st);
    int run(int mode, int group, int disp_mask, int with_update, float lr, float mu, float gscale, cudaStream_t st);
    int run_eager(int mode, int group, int disp_mask, int with_update, float lr, float mu, float gscale, cudaStream_t st);
    // ---- per-layer kernel plan (ConvPlan) and the split-16-bit wgmma path (conv_bf.cu, wgrad_bf.cu)
    std::vector<ConvPlan> plan;                    // per layer, filled by layout()
    void plan_views(int li, const TView& x, const TView& y, const TView& dpre, const TView& dx);
    int plan_convs(Bump& A, size_t& max_wg, size_t& max_wt);
    std::map<const float*, ActPlanes> planes;      // 16-bit hi/lo planes of the tensors BF kernels read (key: base pointer)
    std::set<const float*> fresh;                  // planes already written by a conv epilogue in the current pass
    std::vector<BfPrepJob> bf_jobs; std::vector<int> bf_job_begin, bf_job_end;
    BfPrepJob* bf_jobs_dev; size_t bf_max_total;
    ActPlanes wg_xp; size_t wg_xp_halfs;              // bf16 scratch planes: forward activations re-split for the weight gradient
    float act_scale;                                  // power-of-two scale of the fp16 forward planes (per network)
    int ensure_planes(const TView& v, const ActPlanes* pl, cudaStream_t st);
    void planes_written(const TView& v, const ActPlanes* pl, bool written);
    // kernel arguments of layer li's three directions on its planned views; false: the views do not fit the layer
    bool fwd_args(int li, ConvGemm& p) const;
    bool dgrad_args(int li, ConvGemm& p) const;
    bool wgrad_args(int li, ConvWgrad& q) const;
    int wgrad(const ConvLayer& L, const ConvPlan& P, const ConvWgrad& q, cudaStream_t st);
    // ---- data-parallel exchange over NVLink peer memory (csrc/dp.cu)
    int dp_rank, dp_world; bool dp_connected;
    float* dp_xbuf; DpState* dp_state; size_t dp_cap_floats;
    float* dp_peer_xbuf[DP_MAX_WORLD]; DpState* dp_peer_state[DP_MAX_WORLD];
    int dp_create(int rank, int world, unsigned char* handles_out /* 128 bytes */);
    int dp_connect(const unsigned char* all_handles /* world x 128 bytes */);
    int dp_update(int group, float lr, float mu, cudaStream_t st);
    int dp_error(unsigned int* out);
    float* wg_ws; size_t wg_ws_floats;
    float* rs_tmp; size_t rs_tmp_floats;
    float* loss_ws; size_t loss_ws_floats;
    float* loss_full_ws;             // full-resolution loss without gradient, apart from loss_ws (nullptr: shares loss_ws)
    unsigned char* u8_stage;         // 2 x B*H*W*3 bytes: uint8 input staging (set_input_u8)
    // rectification of set_input_u8_resized (ms_engine_set_rectification): [rect_h,rect_w,2] remap table per camera and a
    // 2 x B*rect_h*rect_w*3 byte scratch for the rectified frames, caller-owned; rect_map_l == nullptr: off
    const float* rect_map_l; const float* rect_map_r;
    int rect_h, rect_w;
    unsigned char* rect_scratch;
    // MAD module losses at 1/rs_scale resolution (ms_engine_set_reprojection_scale, --reprojectionScale); rs_scale 1: full
    // resolution.  Views and tap tables live in the caller's scratch: rs_left / rs_right [B,h,w,3], rs_proxy / rs_disp
    // [B,h,w,1] (h = H / rs_scale, w = W / rs_scale); per module the row / column taps of rs_module_disp and their ranges.  The
    // module loss's gradient [B,h,w] reuses g_disp.  rs_fresh: rs_left / rs_right / rs_proxy hold the current frame's values
    int rs_scale;
    TView rs_left, rs_right, rs_proxy, rs_disp;
    struct RsTables { RsTap *rows, *cols; RsRange *rrange, *crange; };
    RsTables rs_tab[5];
    bool rs_fresh;
    size_t rs_layout(int s, float* base);          // scratch floats; base != nullptr: also place the views and tables
    int reprojection_scratch_floats(int s, size_t* floats);
    int set_reprojection_scale(int s, float* scratch, size_t scratch_floats);
    bool rs_module(int which, int slot) const { return rs_scale > 1 && net == 0 && slot == 1 && which >= 0 && which < 5; }
    int rs_prepare_inputs(cudaStream_t st);
    // optimizer of update(): 0 = momentum SGD (Mo = accumulator), 1 = Adam (Mo = first moment, adam_v = second moment,
    // adam_powers = device [beta1_power, beta2_power] shared by every train op); caller-owned storage (ms_engine_set_optimizer)
    int opt_kind;
    float adam_b1, adam_b2, adam_eps;
    float* adam_v; float* adam_powers;
    float* scalars;                  // [0]=full loss, [1]=train loss, [2]=epe, [3]=bad3
    float* gt;                       // optional ground truth [B,H,W,1]
    float* proxy;                    // proxy disparities [B,H,W,1] of the continual-adaptation variant (loss_kind 1)
    int loss_kind;                   // 0 = reprojection SSIM+L1 (Stereo_Online_Adaptation.py), 1 = masked L1 to proxy labels (Stereo_Continual_Adaptation.py)
    float proxy_w_full, proxy_w_module;   // loss weights of the reference: 0.01 (full-resolution loss / FULL train op), 0.1 (MAD module losses)

    // ---- profiling (off by default): CUDA events around kernel groups on the launching stream
    enum Cat { CAT_CONV_FWD = 0, CAT_CONV_DGRAD, CAT_CONV_WGRAD, CAT_CORR_FWD, CAT_CORR_BWD, CAT_LOSS, CAT_OTHER, N_CAT };
    struct Span { int cat, layer; cudaEvent_t a, b; double macs, bytes; };
    int profiling;                   // 0 off, 1 eager (events between launches), 2 in-graph (external event nodes inside the replayed graph)
    bool prof_capturing;
    float prof_event_overhead_ms;    // in-graph event-to-event latency with nothing in between (calibration)
    std::vector<Span> spans;
    std::vector<cudaEvent_t> event_pool;
    double cat_ms[N_CAT]; double cat_macs[N_CAT]; double cat_bytes[N_CAT]; long long cat_calls[N_CAT];
    void prof_begin(int cat, cudaStream_t st, int layer = -1);
    void prof_end(cudaStream_t st);
    void prof_note(double macs, double bytes);   // work of the span just closed
    int prof_fold(std::vector<Span>& v, bool recycle);
    std::vector<double> layer_ms[3]; std::vector<long long> layer_calls[3];   // per layer: fwd / dgrad / wgrad
    int prof_collect();      // synchronises; folds spans into cat_ms
    void prof_reset();

    // ---- DispNet buffers (engine_dispnet.cu)
    TView d_c1, d_c2, d_cat3, d_enc[8], d_cat[5], d_pr[5], d_cc[5], d_pred;
    TView gd_c1, gd_c2, gd_cat3, gd_enc[8], gd_cat[5], gd_pr[5], gd_cc[5], gd_pred;
    int build_dispnet();
    void layout_dispnet(Bump& A);
    int forward_dispnet(int disp_mask, cudaStream_t st);
    int backward_dispnet(cudaStream_t st);
    int deconv_bwd(int li, int dx_acc, cudaStream_t st);

    Engine();
    // *floats: the workspace floats needed; base == nullptr: sizing only (the views are not usable).  -2: a layer's
    // planned views do not fit it
    int layout(float* base, size_t* floats);
    int build_madnet();
    int finalize_groups(const int* group_of_layer, int n_groups);

    int set_input(const float* left, const float* right, cudaStream_t st);
    int set_input_u8(const unsigned char* left, const unsigned char* right, cudaStream_t st);
    int set_input_u8_resized(const unsigned char* left, const unsigned char* right, int h, int w, int rh, int rw, cudaStream_t st);
    int set_rectification(const float* map_left, const float* map_right, int h, int w, unsigned char* scratch, size_t scratch_bytes);
    int set_optimizer(int kind, float beta1, float beta2, float eps, float* v, float* powers);
    void drop_graphs();
    // branch != nullptr: right after module fork_group's disparity head, `branch` waits for `st`, and that module's
    // full-resolution disparity is resized on `branch`
    int forward(int disp_mask, cudaStream_t st, int fork_group = -1, cudaStream_t branch = nullptr);
    int loss(int which, int with_grad, int slot, float grad_scale, cudaStream_t st);
    int backward(int mode, int group, cudaStream_t st);     // mode 1 = MAD(group), 2 = FULL
    int update(int group, float lr, float mu, float gscale, cudaStream_t st);

    // helpers: layer li on the views its plan holds
    int conv_fwd(int li, const float* res, int res_cs, cudaStream_t st);
    int conv_bwd(int li, int want_dx, float dx_slope, int dx_acc, int want_wgrad, cudaStream_t st);
    bool trainable(int layer, int mode, int group) const;
};

}  // namespace ms
