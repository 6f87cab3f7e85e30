// Direct kernels for the single-channel disparity heads (bandwidth-bound, no tensor cores: N = 1 has no reuse).
//
// Replaces the cuDNN calls behind the linear 3x3 -> 1 convolutions of the reference: estimator `disp-6`
// (Nets/MadNet.py:113-118), `context-7` with the residual add (:160-168), DispNet `predict` / `prediction`
// (Nets/DispNet.py:49-50,143-146), and their input gradients (1 -> cin).  Round 1 ran these through the generic fp32
// gather GEMM; here a pixel's channel vector is one coalesced 128-bit load per lane.
#include <algorithm>

#include "common.cuh"

namespace ms {

// forward: y[p] = act(sum_{tap,c} x[p + tap][c] * w[tap][c] + b) (+ res[p]); 8 lanes per pixel, 4 channels per lane per step
__global__ void __launch_bounds__(256)
conv_head_fwd_kernel(ConvGemm g, size_t npix) {
    pdl_prologue();
    extern __shared__ float w_s[];                       // [taps][C]
    const int C = g.x.c, taps = g.kh * g.kw;
    for (int i = threadIdx.x; i < taps * C; i += blockDim.x) w_s[i] = g.wmat[i];
    __syncthreads();
    const int sub = threadIdx.x & 7;
    const size_t pix = (size_t)blockIdx.x * 32 + (threadIdx.x >> 3);
    const bool live = pix < npix;
    float acc = 0.f;
    if (live) {
        const int W = g.y.w, H = g.y.h;
        const int ox = (int)(pix % W);
        const size_t t = pix / W;
        const int oy = (int)(t % H);
        const size_t img = t / H;
        for (int r = 0; r < g.kh; ++r) {
            const int iy = oy + g.off_y + r * g.step;
            if (iy < 0 || iy >= g.x.h) continue;
            for (int s = 0; s < g.kw; ++s) {
                const int ix = ox + g.off_x + s * g.step;
                if (ix < 0 || ix >= g.x.w) continue;
                const float* xp = g.x.p + ((img * g.x.h + iy) * g.x.w + ix) * g.x.cs;
                const float* wp = w_s + (r * g.kw + s) * C;
                for (int c = sub * 4; c < C; c += 32) {
                    const float4 v = *reinterpret_cast<const float4*>(xp + c);
                    const float4 w = *reinterpret_cast<const float4*>(wp + c);
                    acc = fmaf(v.x, w.x, acc); acc = fmaf(v.y, w.y, acc); acc = fmaf(v.z, w.z, acc); acc = fmaf(v.w, w.w, acc);
                }
            }
        }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (live && sub == 0) {
        float t = acc + (g.bias ? g.bias[0] : 0.f);
        t = fmaxf(g.alpha * t, t);
        if (g.res) t += g.res[pix * g.res_cs];
        float* yp = g.y.p + pix * g.y.cs;
        if (g.accumulate) t += *yp;
        if (g.mask) t *= (g.mask[pix * g.mask_cs] > 0.f) ? 1.f : g.mask_alpha;
        *yp = t;
    }
}

// input gradient of a 1-channel conv: dx[p][c] = sum_tap dy[p + off + tap*step] * w[tap][c]   (then accumulate / mask)
__global__ void __launch_bounds__(256)
conv_head_dgrad_kernel(ConvGemm g, size_t npix) {
    pdl_prologue();
    extern __shared__ float w_s[];                       // [taps][C]
    const int C = g.y.c, taps = g.kh * g.kw, cq = C >> 2;
    for (int i = threadIdx.x; i < taps * C; i += blockDim.x) w_s[i] = g.wmat[i];
    __syncthreads();
    const size_t total = npix * cq;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / cq;
        const int c = (int)(i - pix * cq) * 4;
        const int W = g.y.w, H = g.y.h;
        const int ox = (int)(pix % W);
        const size_t t = pix / W;
        const int oy = (int)(t % H);
        const size_t img = t / H;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < g.kh; ++r) {
            const int iy = oy + g.off_y + r * g.step;
            if (iy < 0 || iy >= g.x.h) continue;
            for (int s = 0; s < g.kw; ++s) {
                const int ix = ox + g.off_x + s * g.step;
                if (ix < 0 || ix >= g.x.w) continue;
                const float d = __ldg(g.x.p + ((img * g.x.h + iy) * g.x.w + ix) * g.x.cs);
                const float4 w = *reinterpret_cast<const float4*>(w_s + (r * g.kw + s) * C + c);
                a.x = fmaf(d, w.x, a.x); a.y = fmaf(d, w.y, a.y); a.z = fmaf(d, w.z, a.z); a.w = fmaf(d, w.w, a.w);
            }
        }
        float* yp = g.y.p + pix * g.y.cs + c;
        if (g.accumulate) { const float4 o = *reinterpret_cast<const float4*>(yp); a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w; }
        if (g.mask) {
            const float4 m = *reinterpret_cast<const float4*>(g.mask + pix * g.mask_cs + c);
            a.x *= m.x > 0.f ? 1.f : g.mask_alpha; a.y *= m.y > 0.f ? 1.f : g.mask_alpha;
            a.z *= m.z > 0.f ? 1.f : g.mask_alpha; a.w *= m.w > 0.f ? 1.f : g.mask_alpha;
        }
        *reinterpret_cast<float4*>(yp) = a;
    }
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// 1 = forward head (y.c == 1), 2 = head dgrad (x.c == 1), 0 = not a head
// single-channel gather (1 -> 1 channel, any generic gather geometry): DispNet's `up_predict` 4x4 stride-2 conv_transpose of
// a disparity map (Nets/DispNet.py:51-53).  One thread per output pixel; the generic fp32 gather GEMM is far too slow for
// this 2 MFLOP operation.
__global__ void __launch_bounds__(256) conv_one_channel_kernel(ConvGemm g, size_t npix) {
    pdl_prologue();
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    const int W = g.y.w, H = g.y.h;
    const int ox = (int)(pix % W);
    const size_t t = pix / W;
    const int oy = (int)(t % H);
    const size_t img = t / H;
    float acc = g.bias ? g.bias[0] : 0.f;
    for (int r = 0; r < g.kh; ++r) {
        int ty = oy * g.mul + g.off_y + r * g.step;
        if (g.div > 1) { if (ty % g.div) continue; ty /= g.div; }
        if (ty < 0 || ty >= g.x.h) continue;
        for (int s = 0; s < g.kw; ++s) {
            int tx = ox * g.mul + g.off_x + s * g.step;
            if (g.div > 1) { if (tx % g.div) continue; tx /= g.div; }
            if (tx < 0 || tx >= g.x.w) continue;
            acc = fmaf(g.x.p[((img * g.x.h + ty) * g.x.w + tx) * g.x.cs], g.wmat[r * g.kw + s], acc);
        }
    }
    acc = fmaxf(g.alpha * acc, acc);
    float* yp = g.y.p + pix * g.y.cs;
    if (g.res) acc += g.res[pix * g.res_cs];
    if (g.accumulate) acc += *yp;
    if (g.mask) acc *= (g.mask[pix * g.mask_cs] > 0.f) ? 1.f : g.mask_alpha;
    *yp = acc;
}
bool conv_one_channel_supported(const ConvGemm& g) { return g.x.c == 1 && g.y.c == 1 && g.x.n == g.y.n && g.alpha <= 1.f && g.alpha >= 0.f; }
int conv_one_channel(const ConvGemm& g, cudaStream_t st) {
    MS_REQUIRE(conv_one_channel_supported(g), "conv_one_channel: not a 1 -> 1 channel gather");
    const size_t npix = g.y.pixels();
    launch_k(conv_one_channel_kernel, dim3((unsigned)cdivz(npix, 256)), dim3(256), 0, st, g, npix);
    return check_launch("conv_one_channel");
}

// weight (+ bias) gradient of a conv with ONE output channel: dw[tap][c] = sum_p x[p * stride - pad + tap * dil][c] * dy[p].
// (DispNet `prediction` 32 -> 1 at 192 x 640, `predict` heads, the 1 -> 1 `up_predict` transposed convs with the big map
// in the x role; MADNet `disp-6` / `context-7`.)  288 ... 16 k outputs reduced over up to 123 k pixels: the generic fp32
// wgrad GEMM pads co = 1 to a 16-wide tile; here G lanes share a pixel (4 channels each), every
// thread keeps its K x K x 4 partial sums in registers over a grid-stride pixel loop, and the CTA folds them in a fixed
// order (deterministic) into one partial vector.
template <int K>
__global__ void __launch_bounds__(256)
conv_head_wgrad_kernel(ConvWgrad q, int gshift, size_t npix, float* __restrict__ part, int vec) {
    pdl_prologue();
    extern __shared__ float hw_s[];                      // [256 / G pixel slots][K*K][G*4]  +  [256] bias partials
    constexpr int TAPS = K * K;
    const int G = 1 << gshift, PP = 256 >> gshift;
    const int C = q.x.c;
    const int cg = threadIdx.x & (G - 1), ps = threadIdx.x >> gshift;
    const int c = cg * 4;
    const int nvalid = max(0, min(4, C - c));
    float acc[TAPS][4];
#pragma unroll
    for (int t = 0; t < TAPS; ++t) { acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f; }
    float bsum = 0.f;
    const int W = q.dy.w, H = q.dy.h;
    for (size_t pix = (size_t)blockIdx.x * PP + ps; pix < npix; pix += (size_t)gridDim.x * PP) {
        const int ox = (int)(pix % W);
        const size_t t0 = pix / W;
        const int oy = (int)(t0 % H);
        const size_t img = t0 / H;
        const float d = __ldg(q.dy.p + pix * q.dy.cs);
        if (cg == 0) bsum += d;
        if (nvalid == 0) continue;
#pragma unroll
        for (int r = 0; r < K; ++r) {
            const int iy = oy * q.stride - q.pad_t + r * q.dil;
            if (iy < 0 || iy >= q.x.h) continue;
#pragma unroll
            for (int s = 0; s < K; ++s) {
                const int ix = ox * q.stride - q.pad_l + s * q.dil;
                if (ix < 0 || ix >= q.x.w) continue;
                const float* xp = q.x.p + ((img * q.x.h + iy) * q.x.w + ix) * q.x.cs + c;
                if (vec) {
                    const float4 v = __ldg(reinterpret_cast<const float4*>(xp));
                    acc[r * K + s][0] = fmaf(v.x, d, acc[r * K + s][0]); acc[r * K + s][1] = fmaf(v.y, d, acc[r * K + s][1]);
                    acc[r * K + s][2] = fmaf(v.z, d, acc[r * K + s][2]); acc[r * K + s][3] = fmaf(v.w, d, acc[r * K + s][3]);
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (j < nvalid) acc[r * K + s][j] = fmaf(__ldg(xp + j), d, acc[r * K + s][j]);
                }
            }
        }
    }
    // fold the pixel slots in slot order
    const int row = TAPS * G * 4;
#pragma unroll
    for (int t = 0; t < TAPS; ++t)
        *reinterpret_cast<float4*>(hw_s + (size_t)ps * row + (t * G + cg) * 4) = make_float4(acc[t][0], acc[t][1], acc[t][2], acc[t][3]);
    float* bs = hw_s + (size_t)PP * row;
    bs[threadIdx.x] = cg == 0 ? bsum : 0.f;
    __syncthreads();
    float* mine = part + (size_t)blockIdx.x * (TAPS * C + 1);
    for (int i = threadIdx.x; i < TAPS * C; i += 256) {
        const int t = i / C, ch = i - t * C;
        float sum = 0.f;
        for (int k = 0; k < PP; ++k) sum += hw_s[(size_t)k * row + t * G * 4 + ch];
        mine[i] = sum;
    }
    if (threadIdx.x == 0) {
        float sum = 0.f;
        for (int k = 0; k < 256; ++k) sum += bs[k];
        mine[TAPS * C] = sum;
    }
}

__global__ void conv_head_wgrad_reduce_kernel(const float* __restrict__ part, int nparts, int n, float* __restrict__ dw,
                                              float* __restrict__ db, int accumulate) {
    pdl_prologue();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    float sum = 0.f;
    for (int k = 0; k < nparts; ++k) sum += part[(size_t)k * (n + 1) + i];
    if (i < n) dw[i] = accumulate ? dw[i] + sum : sum;
    else if (db) db[0] = accumulate ? db[0] + sum : sum;
}

static int head_wgrad_grid(const ConvWgrad& q, int& gshift) {
    const int c4 = (q.x.c + 3) / 4;
    gshift = 0;
    while ((1 << gshift) < c4) ++gshift;
    const size_t pp = 256 >> gshift;
    return (int)std::min<size_t>(cdivz(q.dy.pixels(), pp), 2 * NUM_SMS);
}
bool conv_head_wgrad_supported(const ConvWgrad& q) {
    return q.dy.c == 1 && q.kh == q.kw && (q.kh == 3 || q.kh == 4) && q.x.c >= 1 && q.x.c <= 1024 && q.x.n == q.dy.n;
}
size_t conv_head_wgrad_workspace_floats(const ConvWgrad& q) {
    int gs;
    return (size_t)head_wgrad_grid(q, gs) * ((size_t)q.kh * q.kw * q.x.c + 1);
}
// q.dw: [tap][cin] (= [tap][cin][1]); q.db: [1] or nullptr
int conv_head_wgrad(const ConvWgrad& q, cudaStream_t st) {
    MS_REQUIRE(conv_head_wgrad_supported(q), "conv_head_wgrad: not a single-output-channel weight gradient");
    int gshift;
    const int grid = head_wgrad_grid(q, gshift);
    const int taps = q.kh * q.kw, n = taps * q.x.c;
    MS_REQUIRE(q.workspace_floats >= (size_t)grid * (n + 1), "conv_head_wgrad: workspace too small");
    const size_t smem = (size_t)256 * taps * 16 + 256 * sizeof(float);
    static bool attr_done = false;
    if (!attr_done) {
        MS_CHECK_CUDA(cudaFuncSetAttribute(conv_head_wgrad_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
        MS_CHECK_CUDA(cudaFuncSetAttribute(conv_head_wgrad_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
        attr_done = true;
    }
    const int vec = ((q.x.c & 3) == 0 && (q.x.cs & 3) == 0 && aligned16(q.x.p)) ? 1 : 0;
    const size_t npix = q.dy.pixels();
    if (q.kh == 3) launch_k(conv_head_wgrad_kernel<3>, dim3(grid), dim3(256), smem, st, q, gshift, npix, q.workspace, vec);
    else launch_k(conv_head_wgrad_kernel<4>, dim3(grid), dim3(256), smem, st, q, gshift, npix, q.workspace, vec);
    launch_k(conv_head_wgrad_reduce_kernel, dim3(cdiv(n + 1, 256)), dim3(256), 0, st, (const float*)q.workspace, grid, n, q.dw, q.db, q.accumulate);
    return check_launch("conv_head_wgrad", 2);
}

int conv_head_kind(const ConvGemm& g) {
    if (g.mul != 1 || g.div != 1) return 0;
    if (g.x.h != g.y.h || g.x.w != g.y.w) return 0;
    const size_t wbytes = (size_t)g.kh * g.kw * std::max(g.x.c, g.y.c) * sizeof(float);
    if (wbytes > 96 * 1024) return 0;
    if (g.y.c == 1 && g.x.c >= 4 && (g.x.c & 3) == 0 && (g.x.cs & 3) == 0 && aligned16(g.x.p) && aligned16(g.wmat)) return 1;
    if (g.x.c == 1 && g.y.c >= 4 && (g.y.c & 3) == 0 && (g.y.cs & 3) == 0 && aligned16(g.y.p) && aligned16(g.wmat) && !g.res &&
        !g.bias && g.alpha == 1.f && (!g.mask || ((g.mask_cs & 3) == 0 && aligned16(g.mask))))
        return 2;
    return 0;
}

// g.wmat: [tap][cin] for the forward head, [tap][cin] (= [tap][1][cin]) for its dgrad -- the same memory either way
int conv_head(const ConvGemm& g, cudaStream_t st) {
    const int kind = conv_head_kind(g);
    MS_REQUIRE(kind != 0, "conv_head: not a single-channel head");
    static bool attr_done = false;
    if (!attr_done) {
        MS_CHECK_CUDA(cudaFuncSetAttribute(conv_head_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        MS_CHECK_CUDA(cudaFuncSetAttribute(conv_head_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr_done = true;
    }
    const size_t npix = g.y.pixels();
    const size_t smem = (size_t)g.kh * g.kw * std::max(g.x.c, g.y.c) * sizeof(float);
    if (kind == 1) {
        launch_k(conv_head_fwd_kernel, dim3((unsigned)cdivz(npix, 32)), dim3(256), smem, st, g, npix);
        return check_launch("conv_head_fwd");
    }
    const size_t total = npix * (g.y.c >> 2);
    const unsigned grid = (unsigned)std::min<size_t>(cdivz(total, 256), NUM_SMS * 8);
    launch_k(conv_head_dgrad_kernel, dim3(grid), dim3(256), smem, st, g, npix);
    return check_launch("conv_head_dgrad");
}

}  // namespace ms
