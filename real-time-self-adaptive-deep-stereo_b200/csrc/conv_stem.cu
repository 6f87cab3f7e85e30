// Direct fp32 kernels for DispNet's stem: conv1, 7 x 7 stride 2, 3 -> 64 channels on the full-resolution image pair
// (reference Nets/DispNet.py:82-86 through sharedLayers.conv2d, Nets/sharedLayers.py:54-63) -- forward and the filter
// gradient tf.gradients derives for it in the FULL train op (Stereo_Online_Adaptation.py:118,143-151).
//
// 2.3 GMAC per pass over 2 x 384 x 1280 pixels with a reduction depth of 3 channels: on the swap-AB tensor-core path the
// K block of every tap is 3 real channels in 32 and the weight gradient fills 3 of the 128 accumulator rows.  The CUDA
// cores do the same arithmetic without that padding; what decides is operand reuse in registers:
//   wgrad  : a CTA stages an 8 x 16 output tile (input patch 21 x 37 x 3, dY 128 x 64) in shared memory; a thread owns
//            5 (tap, ci) pairs x 8 output channels = 40 partial sums and reads 5 x + 8 dY values per 40 FMAs; CTAs are
//            persistent over tiles and leave one partial vector each, folded in a fixed order (deterministic).
//   forward: same tile; a thread owns 4 adjacent output pixels x 8 output channels; per filter row the 13 input pixels
//            they touch are held in registers for all 7 horizontal taps (the 147 x 64 filter sits in shared memory).
#include <algorithm>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace ms {

constexpr int ST_K = 7, ST_CI = 3, ST_CO = 64, ST_S = 2;
constexpr int ST_TH = 8, ST_TW = 16;                         // output tile
constexpr int ST_PH = (ST_TH - 1) * ST_S + ST_K;             // 21 patch rows
constexpr int ST_PW = (ST_TW - 1) * ST_S + ST_K;             // 37 patch columns
constexpr int ST_NT = 256;
constexpr int ST_TAPS = ST_K * ST_K * ST_CI;                 // 147 (tap, ci) pairs
constexpr int ST_PER = 5;                                    // pairs per thread: 30 thread groups cover 150 >= 147

static bool stem_geom(int xc, int xcs, int yc, int kh, int kw, int stride, int dil) {
    return xc == ST_CI && xcs == 4 && yc == ST_CO && kh == ST_K && kw == ST_K && stride == ST_S && dil == 1;
}

// stage the input patch (float4 per pixel: 3 channels + the pad lane) of tile (img, ty, tx); zeros outside the image
__device__ __forceinline__ void stem_load_patch(float4* xs, const float* x, int xh, int xw, int img, int iy0, int ix0) {
    for (int e = threadIdx.x; e < ST_PH * ST_PW; e += ST_NT) {
        const int r = e / ST_PW, c = e - r * ST_PW;
        const int iy = iy0 + r, ix = ix0 + c;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (iy >= 0 && iy < xh && ix >= 0 && ix < xw) v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)img * xh + iy) * xw + ix) * 4));
        xs[e] = v;
    }
}

__global__ void __launch_bounds__(ST_NT, 2)
conv_stem_wgrad_kernel(ConvWgrad q, int tiles_x, int tiles_y, int ntiles, float* __restrict__ part) {
    pdl_prologue();
    extern __shared__ __align__(16) unsigned char stem_smem[];
    float4* xs = reinterpret_cast<float4*>(stem_smem);                          // [21][37] pixels x (3 + pad)
    float* dys = reinterpret_cast<float*>(xs + ST_PH * ST_PW);                  // [128][64]
    const int cg = threadIdx.x & 7, tg = threadIdx.x >> 3;                      // 8 output channels; 5 (tap, ci) pairs
    int off[ST_PER];
#pragma unroll
    for (int j = 0; j < ST_PER; ++j) {
        const int e = min(tg * ST_PER + j, ST_TAPS - 1);                   // (the 3 surplus slots recompute pair 146; never stored)
        const int c = e % ST_CI, s = (e / ST_CI) % ST_K, r = e / (ST_CI * ST_K);
        off[j] = (r * ST_PW + s) * 4 + c;
    }
    float acc[ST_PER][8];
#pragma unroll
    for (int j = 0; j < ST_PER; ++j)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[j][k] = 0.f;
    const bool bias_thread = tg == 30;                                          // an otherwise idle group sums dY for the bias
    const float* xsf = reinterpret_cast<const float*>(xs);
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int img = t / (tiles_x * tiles_y);
        const int rem = t - img * tiles_x * tiles_y;
        const int ty = rem / tiles_x, tx = rem - ty * tiles_x;
        const int oy0 = ty * ST_TH, ox0 = tx * ST_TW;
        __syncthreads();                                                        // previous tile consumed
        stem_load_patch(xs, q.x.p, q.x.h, q.x.w, img, oy0 * ST_S - q.pad_t, ox0 * ST_S - q.pad_l);
        for (int e = threadIdx.x; e < ST_TH * ST_TW * (ST_CO / 4); e += ST_NT) {
            const int px = e / (ST_CO / 4), c4 = e - px * (ST_CO / 4);
            const int oy = oy0 + px / ST_TW, ox = ox0 + px % ST_TW;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (oy < q.dy.h && ox < q.dy.w)
                v = __ldg(reinterpret_cast<const float4*>(q.dy.p + (((size_t)img * q.dy.h + oy) * q.dy.w + ox) * q.dy.cs + c4 * 4));
            reinterpret_cast<float4*>(dys)[e] = v;
        }
        __syncthreads();
        if (tg < 30) {
#pragma unroll 2
            for (int px = 0; px < ST_TH * ST_TW; ++px) {
                const int pbase = ((px / ST_TW) * ST_S * ST_PW + (px % ST_TW) * ST_S) * 4;
                const float4 d0 = *reinterpret_cast<const float4*>(dys + px * ST_CO + cg * 8);
                const float4 d1 = *reinterpret_cast<const float4*>(dys + px * ST_CO + cg * 8 + 4);
#pragma unroll
                for (int j = 0; j < ST_PER; ++j) {
                    const float xv = xsf[pbase + off[j]];
                    acc[j][0] = fmaf(xv, d0.x, acc[j][0]); acc[j][1] = fmaf(xv, d0.y, acc[j][1]);
                    acc[j][2] = fmaf(xv, d0.z, acc[j][2]); acc[j][3] = fmaf(xv, d0.w, acc[j][3]);
                    acc[j][4] = fmaf(xv, d1.x, acc[j][4]); acc[j][5] = fmaf(xv, d1.y, acc[j][5]);
                    acc[j][6] = fmaf(xv, d1.z, acc[j][6]); acc[j][7] = fmaf(xv, d1.w, acc[j][7]);
                }
            }
        } else if (bias_thread) {
            for (int px = 0; px < ST_TH * ST_TW; ++px) {
                const float4 d0 = *reinterpret_cast<const float4*>(dys + px * ST_CO + cg * 8);
                const float4 d1 = *reinterpret_cast<const float4*>(dys + px * ST_CO + cg * 8 + 4);
                acc[0][0] += d0.x; acc[0][1] += d0.y; acc[0][2] += d0.z; acc[0][3] += d0.w;
                acc[0][4] += d1.x; acc[0][5] += d1.y; acc[0][6] += d1.z; acc[0][7] += d1.w;
            }
        }
    }
    // partial vector of this CTA: [147][64] weights, then [64] bias sums
    float* mine = part + (size_t)blockIdx.x * (ST_TAPS * ST_CO + ST_CO);
    if (tg < 30) {
#pragma unroll
        for (int j = 0; j < ST_PER; ++j) {
            const int e = tg * ST_PER + j;
            if (e >= ST_TAPS) continue;
            float* dst = mine + (size_t)e * ST_CO + cg * 8;
            *reinterpret_cast<float4*>(dst) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
        }
    } else if (bias_thread) {
        float* dst = mine + (size_t)ST_TAPS * ST_CO + cg * 8;
        *reinterpret_cast<float4*>(dst) = make_float4(acc[0][0], acc[0][1], acc[0][2], acc[0][3]);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[0][4], acc[0][5], acc[0][6], acc[0][7]);
    }
}

// dw[i] = sum over CTAs in index order (i < 147 * 64: [tap][ci][co]); db[c] from the tail of the partial vectors
__global__ void conv_stem_wgrad_reduce_kernel(const float* __restrict__ part, int nparts, float* __restrict__ dw, float* __restrict__ db,
                                              int accumulate) {
    pdl_prologue();
    const int n = ST_TAPS * ST_CO;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n + ST_CO) return;
    float sum = 0.f;
    for (int k = 0; k < nparts; ++k) sum += part[(size_t)k * (n + ST_CO) + i];
    if (i < n) dw[i] = accumulate ? dw[i] + sum : sum;
    else if (db) db[i - n] = accumulate ? db[i - n] + sum : sum;
}

static int stem_wgrad_grid(const ConvWgrad& q) {
    const long ntiles = (long)q.dy.n * cdiv(q.dy.w, ST_TW) * cdiv(q.dy.h, ST_TH);
    return (int)std::min<long>(ntiles, 2 * NUM_SMS);
}
bool conv_stem_wgrad_supported(const ConvWgrad& q) {
    return stem_geom(q.x.c, q.x.cs, q.dy.c, q.kh, q.kw, q.stride, q.dil) && q.x.n == q.dy.n && (q.dy.cs & 3) == 0 &&
           ((reinterpret_cast<uintptr_t>(q.x.p) | reinterpret_cast<uintptr_t>(q.dy.p)) & 15) == 0;
}
size_t conv_stem_wgrad_workspace_floats(const ConvWgrad& q) { return (size_t)stem_wgrad_grid(q) * (ST_TAPS * ST_CO + ST_CO); }
int conv_stem_wgrad(const ConvWgrad& q, cudaStream_t st) {
    MS_REQUIRE(conv_stem_wgrad_supported(q), "conv_stem_wgrad: not the 7x7 stride-2 3 -> 64 stem");
    const int grid = stem_wgrad_grid(q);
    MS_REQUIRE(q.workspace_floats >= conv_stem_wgrad_workspace_floats(q), "conv_stem_wgrad: workspace too small");
    const int tiles_x = cdiv(q.dy.w, ST_TW), tiles_y = cdiv(q.dy.h, ST_TH);
    const size_t smem = (size_t)ST_PH * ST_PW * 16 + (size_t)ST_TH * ST_TW * ST_CO * 4;
    static bool attr = false;
    if (!attr) {
        MS_CHECK_CUDA(cudaFuncSetAttribute(conv_stem_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    launch_k(conv_stem_wgrad_kernel, dim3(grid), dim3(ST_NT), smem, st, q, tiles_x, tiles_y, q.dy.n * tiles_x * tiles_y, q.workspace);
    launch_k(conv_stem_wgrad_reduce_kernel, dim3(cdiv(ST_TAPS * ST_CO + ST_CO, 256)), dim3(256), 0, st, (const float*)q.workspace, grid, q.dw, q.db,
             q.accumulate);
    return check_launch("conv_stem_wgrad", 2);
}

// ---------------------------------------------------------------------------------------------
// forward: y = act(conv(x) + b) (+ 16-bit planes of y for the next layer's tensor-core kernel)
// ---------------------------------------------------------------------------------------------
// x = hi + lo in the plane format of the consumer (same arithmetic as conv_bf.cu:split16): 0 = bf16, 1 = fp16 of x * scale
__device__ __forceinline__ void stem_split16(float v, int fmt, float scale, unsigned short& h, unsigned short& l) {
    if (fmt == 0) {
        const __nv_bfloat16 hb = __float2bfloat16_rn(v);
        h = __bfloat16_as_ushort(hb);
        l = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(hb)));
    } else {
        const float t = v * scale;
        unsigned short hh, ll;
        asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(hh) : "f"(t));
        const float r = t - __half2float(__ushort_as_half(hh));
        asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(ll) : "f"(r));
        h = hh; l = ll;
    }
}

__global__ void __launch_bounds__(ST_NT, 2)
conv_stem_fwd_kernel(ConvGemm g, int tiles_x, int tiles_y, unsigned short* __restrict__ ohi, unsigned short* __restrict__ olo, int ocs,
                     int ofmt, float oscale) {
    pdl_prologue();
    extern __shared__ __align__(16) unsigned char stem_smem[];
    float4* xs = reinterpret_cast<float4*>(stem_smem);                          // [21][37] pixels x (3 + pad)
    float* ws = reinterpret_cast<float*>(xs + ST_PH * ST_PW);                   // [147][64]
    for (int i = threadIdx.x; i < ST_TAPS * ST_CO / 4; i += ST_NT)
        reinterpret_cast<float4*>(ws)[i] = __ldg(reinterpret_cast<const float4*>(g.wmat) + i);
    const int t = blockIdx.x;
    const int img = t / (tiles_x * tiles_y);
    const int rem = t - img * tiles_x * tiles_y;
    const int ty = rem / tiles_x, tx = rem - ty * tiles_x;
    const int oy0 = ty * ST_TH, ox0 = tx * ST_TW;
    stem_load_patch(xs, g.x.p, g.x.h, g.x.w, img, oy0 * ST_S + g.off_y, ox0 * ST_S + g.off_x);
    __syncthreads();
    // thread: 8 output channels (cq) of 4 horizontally adjacent output pixels (pg): 32 pixel groups x 8 channel groups.
    // Per filter row the 13 input pixels the 4 outputs touch (columns 2*px0 ... 2*px0 + 12) sit in registers and serve all
    // 7 horizontal taps: 13 + 42 128-bit shared loads per 672 FMAs.  (First version: 2 pixels x 16 channels, 6 loads per
    // 32 FMAs -- shared-memory bound.)
    const int cq = threadIdx.x & 7, pg = threadIdx.x >> 3;
    const int py = pg / (ST_TW / 4), px = (pg % (ST_TW / 4)) * 4;
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[i][k] = 0.f;
    const float4* xrow0 = xs + (py * ST_S) * ST_PW + px * ST_S;
    for (int r = 0; r < ST_K; ++r) {
        float4 xv[13];
#pragma unroll
        for (int c = 0; c < 13; ++c) xv[c] = xrow0[r * ST_PW + c];
#pragma unroll
        for (int s = 0; s < ST_K; ++s) {
#pragma unroll
            for (int c = 0; c < ST_CI; ++c) {
                const float4* w4 = reinterpret_cast<const float4*>(ws + ((r * ST_K + s) * ST_CI + c) * ST_CO + cq * 8);
                const float4 w0 = w4[0], w1 = w4[1];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float4 xp = xv[2 * i + s];
                    const float x = c == 0 ? xp.x : (c == 1 ? xp.y : xp.z);
                    acc[i][0] = fmaf(x, w0.x, acc[i][0]); acc[i][1] = fmaf(x, w0.y, acc[i][1]);
                    acc[i][2] = fmaf(x, w0.z, acc[i][2]); acc[i][3] = fmaf(x, w0.w, acc[i][3]);
                    acc[i][4] = fmaf(x, w1.x, acc[i][4]); acc[i][5] = fmaf(x, w1.y, acc[i][5]);
                    acc[i][6] = fmaf(x, w1.z, acc[i][6]); acc[i][7] = fmaf(x, w1.w, acc[i][7]);
                }
            }
        }
    }
    const int oy = oy0 + py;
    if (oy >= g.y.h) return;
    float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
    if (g.bias) { b0 = __ldg(reinterpret_cast<const float4*>(g.bias + cq * 8)); b1 = __ldg(reinterpret_cast<const float4*>(g.bias + cq * 8 + 4)); }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int ox = ox0 + px + i;
        if (ox >= g.y.w) continue;
        const size_t pix = ((size_t)img * g.y.h + oy) * g.y.w + ox;
        float* yp = g.y.p + pix * g.y.cs + cq * 8;
        float4 v0 = make_float4(acc[i][0] + b0.x, acc[i][1] + b0.y, acc[i][2] + b0.z, acc[i][3] + b0.w);
        float4 v1 = make_float4(acc[i][4] + b1.x, acc[i][5] + b1.y, acc[i][6] + b1.z, acc[i][7] + b1.w);
        v0.x = fmaxf(g.alpha * v0.x, v0.x); v0.y = fmaxf(g.alpha * v0.y, v0.y); v0.z = fmaxf(g.alpha * v0.z, v0.z); v0.w = fmaxf(g.alpha * v0.w, v0.w);
        v1.x = fmaxf(g.alpha * v1.x, v1.x); v1.y = fmaxf(g.alpha * v1.y, v1.y); v1.z = fmaxf(g.alpha * v1.z, v1.z); v1.w = fmaxf(g.alpha * v1.w, v1.w);
        *reinterpret_cast<float4*>(yp) = v0;
        *reinterpret_cast<float4*>(yp + 4) = v1;
        if (ohi) {
            unsigned short h[8], l[8];
            stem_split16(v0.x, ofmt, oscale, h[0], l[0]); stem_split16(v0.y, ofmt, oscale, h[1], l[1]);
            stem_split16(v0.z, ofmt, oscale, h[2], l[2]); stem_split16(v0.w, ofmt, oscale, h[3], l[3]);
            stem_split16(v1.x, ofmt, oscale, h[4], l[4]); stem_split16(v1.y, ofmt, oscale, h[5], l[5]);
            stem_split16(v1.z, ofmt, oscale, h[6], l[6]); stem_split16(v1.w, ofmt, oscale, h[7], l[7]);
            uint4 hv, lv;
            hv.x = (uint32_t)h[0] | ((uint32_t)h[1] << 16); hv.y = (uint32_t)h[2] | ((uint32_t)h[3] << 16);
            hv.z = (uint32_t)h[4] | ((uint32_t)h[5] << 16); hv.w = (uint32_t)h[6] | ((uint32_t)h[7] << 16);
            lv.x = (uint32_t)l[0] | ((uint32_t)l[1] << 16); lv.y = (uint32_t)l[2] | ((uint32_t)l[3] << 16);
            lv.z = (uint32_t)l[4] | ((uint32_t)l[5] << 16); lv.w = (uint32_t)l[6] | ((uint32_t)l[7] << 16);
            *reinterpret_cast<uint4*>(ohi + pix * ocs + cq * 8) = hv;
            *reinterpret_cast<uint4*>(olo + pix * ocs + cq * 8) = lv;
        }
    }
}

bool conv_stem_fwd_supported(const ConvGemm& g) {
    return g.div == 1 && stem_geom(g.x.c, g.x.cs, g.y.c, g.kh, g.kw, g.mul, g.step) && g.x.n == g.y.n && !g.res && !g.mask && !g.accumulate &&
           (g.y.cs & 3) == 0 &&
           ((reinterpret_cast<uintptr_t>(g.x.p) | reinterpret_cast<uintptr_t>(g.y.p) | reinterpret_cast<uintptr_t>(g.wmat)) & 15) == 0;
}
// g.wmat: canonical HWIO [7][7][3][64]; yp: optional 16-bit planes of y written by the epilogue
int conv_stem_fwd(const ConvGemm& g, const ActPlanes* yp, cudaStream_t st) {
    MS_REQUIRE(conv_stem_fwd_supported(g), "conv_stem_fwd: not the 7x7 stride-2 3 -> 64 stem");
    const int tiles_x = cdiv(g.y.w, ST_TW), tiles_y = cdiv(g.y.h, ST_TH);
    const size_t smem = (size_t)ST_PH * ST_PW * 16 + (size_t)ST_TAPS * ST_CO * 4;
    static bool attr = false;
    if (!attr) {
        MS_CHECK_CUDA(cudaFuncSetAttribute(conv_stem_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    unsigned short *ohi = nullptr, *olo = nullptr;
    int ocs = 0, ofmt = 0; float oscale = 1.f;
    if (yp && yp->hi) {
        MS_REQUIRE(yp->cs >= ST_CO && (yp->cs & 7) == 0, "conv_stem_fwd: bad output planes");
        ohi = reinterpret_cast<unsigned short*>(yp->hi); olo = reinterpret_cast<unsigned short*>(yp->lo);
        ocs = yp->cs; ofmt = yp->fmt; oscale = yp->fmt == 1 ? yp->scale : 1.f;
    }
    launch_k(conv_stem_fwd_kernel, dim3(g.y.n * tiles_x * tiles_y), dim3(ST_NT), smem, st, g, tiles_x, tiles_y, ohi, olo, ocs, ofmt, oscale);
    return check_launch("conv_stem_fwd");
}

}  // namespace ms
