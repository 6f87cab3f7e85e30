// Resampling / elementwise kernels of the hot path (all HBM-bound, one pass each).
//
//   pad_reflect          preprocessing.pad_image                 (reference Data_utils/preprocessing.py:7-29)
//   resize_bilinear      tf.image.resize_images legacy bilinear  (Nets/MadNet.py:69,274,293,312,331,362;
//                        + resize_image_with_crop_or_pad centre crop, MadNet.py:70,363) with the
//                        relu / x20 / x(-20) scalings of MadNet._make_disp fused in
//   resize_bilinear_bwd  its transpose (what tf.gradients builds), separable two-pass gather => deterministic
//   leaky_bwd            gradient of tf.maximum(alpha*x, x)      (Nets/MadNet.py:366-367)
//   rs_inputs / rs_module_disp / rs_module_disp_bwd
//                        MAD module losses at 1/s resolution (--reprojectionScale, Stereo_Online_Adaptation.py:22-23,
//                        91-107; Stereo_Continual_Adaptation.py:95-112)
#include <algorithm>
#include "common.cuh"

namespace ms {

__device__ __forceinline__ int reflect_idx(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * (n - 1) - i;
    return i;
}

__global__ void pad_reflect_kernel(const float* __restrict__ src, int B, int H, int W, int C,
                                   float* __restrict__ dst, int Hp, int Wp, int dcs, float scale, float bias) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)B * Hp * Wp;
    if (i >= total) return;
    int x = (int)(i % Wp);
    size_t q = i / Wp;
    int y = (int)(q % Hp);
    int b = (int)(q / Hp);
    int pt = (Hp - H) / 2, pl = (Wp - W) / 2;
    int sy = reflect_idx(y - pt, H), sx = reflect_idx(x - pl, W);
    const float* s = src + ((size_t)(b * H + sy) * W + sx) * C;
    float* d = dst + i * dcs;
    for (int c = 0; c < C; ++c) d[c] = s[c] * scale + bias;
    for (int c = C; c < dcs; ++c) d[c] = 0.f;
}

int pad_reflect(const float* src, int B, int H, int W, int C, float* dst, int Hp, int Wp, int dcs,
                float scale, float bias, cudaStream_t st) {
    MS_REQUIRE(Hp - H < 2 * H && Wp - W < 2 * W, "pad_reflect: pad larger than image");
    size_t total = (size_t)B * Hp * Wp;
    launch_k(pad_reflect_kernel, dim3((unsigned)cdivz(total, 256)), dim3(256), 0, st, src, B, H, W, C, dst, Hp, Wp, dcs, scale, bias);
    return check_launch("pad_reflect");
}

struct Lerp { int i0, i1; float f; };
__host__ __device__ __forceinline__ Lerp lerp_coeff(int o, float scale, int in_size) {
    // TF 1.x legacy bilinear: src = dst*scale, no half-pixel centres (on the host: the tap tables of rs_axis_taps)
    float s = (float)o * scale;
    float fl = floorf(s);
    Lerp l;
    l.i0 = (int)fl;
    l.i1 = min(l.i0 + 1, in_size - 1);
    l.f = s - fl;
    return l;
}

__device__ __forceinline__ float pre_op(float v, float sc, int relu) {
    v *= sc;
    return relu ? fmaxf(v, 0.f) : v;
}

__device__ __forceinline__ float resize_at(const float* __restrict__ sb, int scs, int iw, Lerp ly, Lerp lx,
                                           float pre_scale, int pre_relu) {
    float tl = pre_op(sb[((size_t)ly.i0 * iw + lx.i0) * scs], pre_scale, pre_relu);
    float tr = pre_op(sb[((size_t)ly.i0 * iw + lx.i1) * scs], pre_scale, pre_relu);
    float bl = pre_op(sb[((size_t)ly.i1 * iw + lx.i0) * scs], pre_scale, pre_relu);
    float br = pre_op(sb[((size_t)ly.i1 * iw + lx.i1) * scs], pre_scale, pre_relu);
    float top = tl + (tr - tl) * lx.f;
    float bot = bl + (br - bl) * lx.f;
    return top + (bot - top) * ly.f;
}

__global__ void resize_kernel(const float* __restrict__ src, int scs, int B, int ih, int iw,
                              float* __restrict__ dst, int dcs, int rh, int rw, int oh, int ow,
                              float ys, float xs, float pre_scale, int pre_relu, float post_scale, int post_relu) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)B * oh * ow;
    if (i >= total) return;
    int ox = (int)(i % ow);
    size_t q = i / ow;
    int oy = (int)(q % oh);
    int b = (int)(q / oh);
    int cy = (rh - oh) / 2, cx = (rw - ow) / 2;
    Lerp ly = lerp_coeff(oy + cy, ys, ih), lx = lerp_coeff(ox + cx, xs, iw);
    float v = resize_at(src + (size_t)b * ih * iw * scs, scs, iw, ly, lx, pre_scale, pre_relu) * post_scale;
    if (post_relu) v = fmaxf(v, 0.f);
    dst[i * dcs] = v;
}

int resize_bilinear(const float* src, int scs, int B, int ih, int iw, float* dst, int dcs, int rh, int rw,
                    int oh, int ow, float pre_scale, int pre_relu, float post_scale, int post_relu,
                    cudaStream_t st) {
    MS_REQUIRE(oh <= rh && ow <= rw, "resize_bilinear: only centre-crop (no pad) is supported");
    size_t total = (size_t)B * oh * ow;
    float ys = (float)ih / (float)rh, xs = (float)iw / (float)rw;
    launch_k(resize_kernel, dim3((unsigned)cdivz(total, 256)), dim3(256), 0, st, src, scs, B, ih, iw, dst, dcs, rh, rw, oh, ow, ys, xs,
                                                              pre_scale, pre_relu, post_scale, post_relu);
    return check_launch("resize_bilinear");
}

// pass 1: tmp[b, oy, ix] = sum_ox dpost[b,oy,ox] * wx(ox -> ix)            (dpost includes post-relu mask)
__global__ void resize_bwd_x_kernel(const float* __restrict__ dout, int docs, const float* __restrict__ src,
                                    int scs, int B, int ih, int iw, float* __restrict__ tmp, int rh, int rw,
                                    int oh, int ow, float ys, float xs, float pre_scale, int pre_relu,
                                    float post_scale, int post_relu) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)B * oh * iw;
    if (i >= total) return;
    int ix = (int)(i % iw);
    size_t q = i / iw;
    int oy = (int)(q % oh);
    int b = (int)(q / oh);
    int cy = (rh - oh) / 2, cx = (rw - ow) / 2;
    // candidate resized columns X whose taps can touch ix: X*xs in (ix-1, ix+1)
    float inv = (float)rw / (float)iw;
    int Xlo = max(cx, (int)floorf((float)(ix - 1) * inv) - 1);
    int Xhi = min(cx + ow - 1, (int)ceilf((float)(ix + 1) * inv) + 1);
    Lerp ly = lerp_coeff(oy + cy, ys, ih);
    const float* sb = src + (size_t)b * ih * iw * scs;
    float acc = 0.f;
    for (int X = Xlo; X <= Xhi; ++X) {
        Lerp lx = lerp_coeff(X, xs, iw);
        float wgt = 0.f;
        if (lx.i0 == ix) wgt += 1.f - lx.f;
        if (lx.i1 == ix) wgt += lx.f;
        if (wgt == 0.f) continue;
        float g = dout[((size_t)(b * oh + oy) * ow + (X - cx)) * docs] * post_scale;
        if (post_relu) {
            float v = resize_at(sb, scs, iw, ly, lx, pre_scale, pre_relu) * post_scale;
            if (!(v > 0.f)) g = 0.f;
        }
        acc += g * wgt;
    }
    tmp[i] = acc;
}

// pass 2: dsrc[b, iy, ix] (+)= pre'(src) * sum_oy tmp[b,oy,ix] * wy(oy -> iy)
__global__ void resize_bwd_y_kernel(const float* __restrict__ tmp, const float* __restrict__ src, int scs, int B,
                                    int ih, int iw, float* __restrict__ dsrc, int dscs, int rh, int oh, float ys,
                                    float pre_scale, int pre_relu, int accumulate) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)B * ih * iw;
    if (i >= total) return;
    int ix = (int)(i % iw);
    size_t q = i / iw;
    int iy = (int)(q % ih);
    int b = (int)(q / ih);
    int cy = (rh - oh) / 2;
    float inv = (float)rh / (float)ih;
    int Ylo = max(cy, (int)floorf((float)(iy - 1) * inv) - 1);
    int Yhi = min(cy + oh - 1, (int)ceilf((float)(iy + 1) * inv) + 1);
    float acc = 0.f;
    for (int Y = Ylo; Y <= Yhi; ++Y) {
        Lerp ly = lerp_coeff(Y, ys, ih);
        float wgt = 0.f;
        if (ly.i0 == iy) wgt += 1.f - ly.f;
        if (ly.i1 == iy) wgt += ly.f;
        if (wgt == 0.f) continue;
        acc += tmp[((size_t)(b * oh + (Y - cy))) * iw + ix] * wgt;
    }
    float s = src[i * scs];
    float d = pre_scale;
    if (pre_relu && !(s * pre_scale > 0.f)) d = 0.f;
    acc *= d;
    if (accumulate) acc += dsrc[i * dscs];
    dsrc[i * dscs] = acc;
}

// NOTE: the x-pass distributes over the lerp in y only when the pre-op is applied per source tap, which it
// is (pre_op acts on taps, the bilinear mix is linear in the taps), so the separable form is exact.
int resize_bilinear_bwd(const float* dout, int docs, const float* src, int scs, int B, int ih, int iw,
                        float* dsrc, int dscs, int rh, int rw, int oh, int ow, float pre_scale,
                        int pre_relu, float post_scale, int post_relu, int accumulate, float* tmp,
                        cudaStream_t st) {
    MS_REQUIRE(oh <= rh && ow <= rw, "resize_bilinear_bwd: only centre-crop is supported");
    MS_REQUIRE(tmp != nullptr, "resize_bilinear_bwd: tmp workspace (B*oh*iw floats) required");
    float ys = (float)ih / (float)rh, xs = (float)iw / (float)rw;
    size_t t1 = (size_t)B * oh * iw;
    launch_k(resize_bwd_x_kernel, dim3((unsigned)cdivz(t1, 256)), dim3(256), 0, st, dout, docs, src, scs, B, ih, iw, tmp, rh, rw, oh, ow,
                                                                 ys, xs, pre_scale, pre_relu, post_scale, post_relu);
    size_t t2 = (size_t)B * ih * iw;
    launch_k(resize_bwd_y_kernel, dim3((unsigned)cdivz(t2, 256)), dim3(256), 0, st, tmp, src, scs, B, ih, iw, dsrc, dscs, rh, oh, ys,
                                                                 pre_scale, pre_relu, accumulate);
    return check_launch("resize_bilinear_bwd", 2);
}

// ---- MAD module losses at 1/s resolution.  The reference rescales the images with preprocessing.rescale_image (legacy
// bilinear to (H//s, W//s)) and each module disparity -- already at full resolution, crop(resize(relu(-20 V), Hp x Wp))
// -- with resize_to_prediction to the same size.

// left_s / right_s (and proxy_s = resize(proxy) / s) of every frame in one pass: one thread per loss-resolution pixel
__global__ void rs_inputs_kernel(const float* __restrict__ left, const float* __restrict__ right,
                                 const float* __restrict__ proxy, int B, int H, int W, float* __restrict__ dl,
                                 float* __restrict__ dr, float* __restrict__ dp, int h, int w, float ys, float xs, float s) {
    pdl_prologue();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * h * w) return;
    const int x = (int)(i % w);
    const size_t q = i / w;
    const int y = (int)(q % h), b = (int)(q / h);
    const Lerp ly = lerp_coeff(y, ys, H), lx = lerp_coeff(x, xs, W);
    const size_t off = (size_t)b * H * W;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        dl[i * 3 + c] = resize_at(left + off * 3 + c, 3, W, ly, lx, 1.f, 0);
        dr[i * 3 + c] = resize_at(right + off * 3 + c, 3, W, ly, lx, 1.f, 0);
    }
    if (dp) dp[i] = resize_at(proxy + off, 1, W, ly, lx, 1.f, 0) / s;      // (a division, as the reference's `/ scale`)
}

int rs_inputs(const float* left, const float* right, const float* proxy, int B, int H, int W, float* dst_left,
              float* dst_right, float* dst_proxy, int h, int w, int s, cudaStream_t st) {
    MS_REQUIRE(B >= 1 && h >= 1 && w >= 1 && h <= H && w <= W && s >= 1, "rs_inputs: bad geometry");
    MS_REQUIRE(!proxy == !dst_proxy, "rs_inputs: the proxy needs an output and the output a proxy");
    const size_t total = (size_t)B * h * w;
    launch_k(rs_inputs_kernel, dim3((unsigned)cdivz(total, 256)), dim3(256), 0, st, left, right, proxy, B, H, W, dst_left,
             dst_right, dst_proxy, h, w, (float)H / (float)h, (float)W / (float)w, (float)s);
    return check_launch("rs_inputs");
}

// One axis of the two resizes as one operator: legacy bilinear in -> r of the pre-op'd source, centre crop to o, legacy
// bilinear o -> n.  taps[j]: the 4 source indices and weights of output j (a clamped or shared index may repeat);
// range[i]: the outputs whose taps name source i (lo > hi: none), what the gather of the adjoint walks.
void rs_axis_taps(int in, int r, int o, int n, RsTap* taps, RsRange* range) {
    const float s1 = (float)in / (float)r, s2 = (float)o / (float)n;
    const int c = (r - o) / 2;
    for (int i = 0; i < in; ++i) range[i] = RsRange{n, -1};
    for (int j = 0; j < n; ++j) {
        const Lerp l2 = lerp_coeff(j, s2, o);
        const int mid[2] = {l2.i0, l2.i1};
        const double w2[2] = {1.0 - (double)l2.f, (double)l2.f};
        for (int a = 0; a < 2; ++a) {
            const Lerp l1 = lerp_coeff(mid[a] + c, s1, in);
            taps[j].i[2 * a] = l1.i0; taps[j].w[2 * a] = (float)(w2[a] * (1.0 - (double)l1.f));
            taps[j].i[2 * a + 1] = l1.i1; taps[j].w[2 * a + 1] = (float)(w2[a] * (double)l1.f);
        }
        for (int t = 0; t < 4; ++t) {
            RsRange& g = range[taps[j].i[t]];
            g.lo = std::min(g.lo, j); g.hi = std::max(g.hi, j);
        }
    }
}

// rs_module_disp: dst[b,y,x] = sum_a rows[y].w[a] * sum_c cols[x].w[c] * relu(pre_scale * src[b, rows[y].i[a], cols[x].i[c]]): both
// resizes composed in registers, no full-resolution map
__global__ void rs_disp_kernel(const float* __restrict__ src, int scs, int B, int ih, int iw, const RsTap* __restrict__ rows,
                               const RsTap* __restrict__ cols, float* __restrict__ dst, int h, int w, float pre_scale) {
    pdl_prologue();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * h * w) return;
    const int x = (int)(i % w);
    const size_t q = i / w;
    const int y = (int)(q % h), b = (int)(q / h);
    const float* sb = src + (size_t)b * ih * iw * scs;
    const RsTap ty = rows[y], tx = cols[x];
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const float* sr = sb + (size_t)ty.i[a] * iw * scs;
        float r = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) r += tx.w[c] * pre_op(sr[(size_t)tx.i[c] * scs], pre_scale, 1);
        acc += ty.w[a] * r;
    }
    dst[i] = acc;
}

int rs_module_disp(const float* src, int scs, int B, int ih, int iw, const RsTap* rows, const RsTap* cols, float* dst, int h, int w,
            float pre_scale, cudaStream_t st) {
    MS_REQUIRE(rows && cols && B >= 1 && h >= 1 && w >= 1, "rs_module_disp: bad arguments");
    const size_t total = (size_t)B * h * w;
    launch_k(rs_disp_kernel, dim3((unsigned)cdivz(total, 256)), dim3(256), 0, st, src, scs, B, ih, iw, rows, cols, dst, h, w,
             pre_scale);
    return check_launch("rs_module_disp");
}

// adjoint of rs_module_disp, x pass: tmp[b,y,ix] = sum over the outputs x that name ix of dout[b,y,x] * (its weights on ix)
__global__ void rs_disp_bwd_x_kernel(const float* __restrict__ dout, const RsTap* __restrict__ cols,
                                     const RsRange* __restrict__ crange, int B, int h, int w, int iw, float* __restrict__ tmp) {
    pdl_prologue();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * h * iw) return;
    const int ix = (int)(i % iw);
    const float* g = dout + (i / iw) * w;
    const RsRange rg = crange[ix];
    float acc = 0.f;
    for (int x = rg.lo; x <= rg.hi; ++x) {
        const RsTap t = cols[x];
        float wgt = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) if (t.i[c] == ix) wgt += t.w[c];
        acc += g[x] * wgt;
    }
    tmp[i] = acc;
}

// y pass: dsrc[b,iy,ix] = relu'(pre_scale * src) * pre_scale * sum over the outputs y that name iy of tmp * (weights)
__global__ void rs_disp_bwd_y_kernel(const float* __restrict__ tmp, const RsTap* __restrict__ rows,
                                     const RsRange* __restrict__ rrange, const float* __restrict__ src, int scs, int B, int ih,
                                     int iw, int h, float* __restrict__ dsrc, int dscs, float pre_scale) {
    pdl_prologue();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * ih * iw) return;
    const int ix = (int)(i % iw);
    const size_t q = i / iw;
    const int iy = (int)(q % ih), b = (int)(q / ih);
    const RsRange rg = rrange[iy];
    float acc = 0.f;
    for (int y = rg.lo; y <= rg.hi; ++y) {
        const RsTap t = rows[y];
        float wgt = 0.f;
#pragma unroll
        for (int a = 0; a < 4; ++a) if (t.i[a] == iy) wgt += t.w[a];
        acc += tmp[((size_t)b * h + y) * iw + ix] * wgt;
    }
    const float d = src[i * scs] * pre_scale > 0.f ? pre_scale : 0.f;
    dsrc[i * dscs] = acc * d;
}

int rs_module_disp_bwd(const float* dout, const float* src, int scs, int B, int ih, int iw, const RsTap* rows, const RsRange* rrange,
                const RsTap* cols, const RsRange* crange, int h, int w, float* dsrc, int dscs, float pre_scale, float* tmp,
                cudaStream_t st) {
    MS_REQUIRE(rows && rrange && cols && crange && tmp && B >= 1 && h >= 1 && w >= 1, "rs_module_disp_bwd: bad arguments");
    const size_t t1 = (size_t)B * h * iw;
    launch_k(rs_disp_bwd_x_kernel, dim3((unsigned)cdivz(t1, 256)), dim3(256), 0, st, dout, cols, crange, B, h, w, iw, tmp);
    const size_t t2 = (size_t)B * ih * iw;
    launch_k(rs_disp_bwd_y_kernel, dim3((unsigned)cdivz(t2, 256)), dim3(256), 0, st, tmp, rows, rrange, src, scs, B, ih, iw, h,
             dsrc, dscs, pre_scale);
    return check_launch("rs_module_disp_bwd", 2);
}

__global__ void leaky_bwd_kernel(float* __restrict__ g, int gcs, const float* __restrict__ act, int acs,
                                 size_t pixels, int c, float alpha) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pixels * c) return;
    size_t p = i / c;
    int ch = (int)(i - p * c);
    if (!(act[p * acs + ch] > 0.f)) g[p * gcs + ch] *= alpha;
}

int leaky_bwd(float* g, int gcs, const float* act, int acs, size_t pixels, int c, float alpha, cudaStream_t st) {
    launch_k(leaky_bwd_kernel, dim3((unsigned)cdivz(pixels * c, 256)), dim3(256), 0, st, g, gcs, act, acs, pixels, c, alpha);
    return check_launch("leaky_bwd");
}

__global__ void add_channels_kernel(float* __restrict__ dst, int dcs, const float* __restrict__ src, int scs,
                                    size_t pixels, int c, float scale, int accumulate) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pixels * c) return;
    size_t p = i / c;
    int ch = (int)(i - p * c);
    float v = src[p * scs + ch] * scale;
    if (accumulate) v += dst[p * dcs + ch];
    dst[p * dcs + ch] = v;
}

int add_channels(float* dst, int dcs, const float* src, int scs, size_t pixels, int c, float scale,
                 int accumulate, cudaStream_t st) {
    launch_k(add_channels_kernel, dim3((unsigned)cdivz(pixels * c, 256)), dim3(256), 0, st, dst, dcs, src, scs, pixels, c, scale, accumulate);
    return check_launch("add_channels");
}

__global__ void fill_kernel(float* p, size_t n, float v) {
    pdl_prologue();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
int fill(float* p, size_t n, float v, cudaStream_t st) {
    if (n == 0) return 0;
    launch_k(fill_kernel, dim3((unsigned)cdivz(n, 256)), dim3(256), 0, st, p, n, v);
    return check_launch("fill");
}

// uint8 image -> fp32 (what tf.image.decode_* + tf.cast do in the reference input pipeline, Data_utils/data_reader.py).
// Four elements per uchar4 load; the last n % 4 elements (e.g. a 1242x375 KITTI frame: 1397250 bytes) are converted one
// by one by the first threads of the grid.
__global__ void u8_to_f32_kernel(const unsigned char* __restrict__ src, float* __restrict__ dst, size_t n) {
    pdl_prologue();
    const size_t n4 = n / 4;
    const uchar4* s4 = reinterpret_cast<const uchar4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = t; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const uchar4 v = s4[i];
        d4[i] = make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
    }
    if (t < (n & 3)) dst[n4 * 4 + t] = (float)src[n4 * 4 + t];
}
int u8_to_f32(const unsigned char* src, float* dst, size_t n, cudaStream_t st) {
    MS_REQUIRE((reinterpret_cast<uintptr_t>(src) & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0, "u8_to_f32: alignment");
    if (n == 0) return 0;
    launch_k(u8_to_f32_kernel, dim3((unsigned)std::min<size_t>(cdivz(n / 4 + 1, 256), NUM_SMS * 8)), dim3(256), 0, st, src, dst, n);
    return check_launch("u8_to_f32");
}

// Camera frames of any size -> the engine's fp32 input, as the live demo builds it (reference Demo/demo_model.py:80-86):
// preprocessing.rescale_image = tf.image.resize_images legacy bilinear to (rh, rw), then
// tf.image.resize_image_with_crop_or_pad to (H, W) -- per axis a centre crop at offset floor((r - H) / 2) or a zero pad of
// floor((H - r) / 2) before.  One thread per output pixel of either frame (left: first B*H*W threads); the result stays
// fp32 (the demo's loss sees the interpolated values).  rh, rw == h, w is exact: every lerp weight is 0.
__global__ void u8_resize_crop_kernel(const unsigned char* __restrict__ left, const unsigned char* __restrict__ right, int B,
                                      int h, int w, int rh, int rw, int oy0, int ox0, float ys, float xs,
                                      float* __restrict__ dl, float* __restrict__ dr, int H, int W) {
    pdl_prologue();
    const size_t per = (size_t)B * H * W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * per) return;
    const bool is_r = i >= per;
    const size_t j = is_r ? i - per : i;
    const int x = (int)(j % W);
    const size_t q = j / W;
    const int y = (int)(q % H), b = (int)(q / H);
    float* d = (is_r ? dr : dl) + j * 3;
    const int ry = y + oy0, rx = x + ox0;
    if (ry < 0 || ry >= rh || rx < 0 || rx >= rw) { d[0] = 0.f; d[1] = 0.f; d[2] = 0.f; return; }
    const unsigned char* s = (is_r ? right : left) + (size_t)b * h * w * 3;
    const Lerp ly = lerp_coeff(ry, ys, h), lx = lerp_coeff(rx, xs, w);
    const unsigned char* t0 = s + ((size_t)ly.i0 * w) * 3;
    const unsigned char* t1 = s + ((size_t)ly.i1 * w) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float tl = t0[lx.i0 * 3 + c], tr = t0[lx.i1 * 3 + c];
        const float bl = t1[lx.i0 * 3 + c], br = t1[lx.i1 * 3 + c];
        const float top = tl + (tr - tl) * lx.f;
        const float bot = bl + (br - bl) * lx.f;
        d[c] = top + (bot - top) * ly.f;
    }
}

int u8_resize_crop(const unsigned char* left, const unsigned char* right, int B, int h, int w, int rh, int rw, float* dst_left,
                   float* dst_right, int H, int W, cudaStream_t st) {
    MS_REQUIRE(B >= 1 && h >= 1 && w >= 1 && rh >= 1 && rw >= 1 && H >= 1 && W >= 1, "u8_resize_crop: bad geometry");
    MS_REQUIRE(left && right && dst_left && dst_right, "u8_resize_crop: null pointer");
    const int oy0 = rh >= H ? (rh - H) / 2 : -((H - rh) / 2);
    const int ox0 = rw >= W ? (rw - W) / 2 : -((W - rw) / 2);
    const float ys = (float)h / (float)rh, xs = (float)w / (float)rw;     // TF: in / out in fp32, src = dst * scale
    const size_t total = 2 * (size_t)B * H * W;
    launch_k(u8_resize_crop_kernel, dim3((unsigned)cdivz(total, 256)), dim3(256), 0, st, left, right, B, h, w, rh, rw, oy0, ox0,
             ys, xs, dst_left, dst_right, H, W);
    return check_launch("u8_resize_crop");
}

// Stereo rectification of raw camera frames, what cv2.remap(frame, map, INTER_LINEAR, BORDER_CONSTANT 0) does, with the
// taps blended in fp32 instead of OpenCV's 1/32-pixel fixed point.  map[y, x] = (src_x, src_y), [h,w,2] float32 (the
// tables of cv2.initUndistortRectifyMap(..., CV_32FC1) stacked), one per camera and shared by the frames of a batch.
// A tap outside the frame reads 0; the blend is rounded to nearest, ties to even, as saturate_cast<uchar> does.  A map
// entry that is NaN or outside [-1, w] x [-1, h] gives 0 without forming an index (every tap of such an entry would be
// outside anyway).  One thread per output pixel of either frame (left: first B*h*w threads; ncam 1 = left only).
__global__ void rectify_u8_kernel(const unsigned char* __restrict__ left, const unsigned char* __restrict__ right,
                                  const float2* __restrict__ map_l, const float2* __restrict__ map_r, int ncam, int B,
                                  int h, int w, unsigned char* __restrict__ dl, unsigned char* __restrict__ dr) {
    pdl_prologue();
    const size_t hw = (size_t)h * w, per = (size_t)B * hw;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)ncam * per) return;
    const bool is_r = i >= per;
    const size_t j = is_r ? i - per : i;
    const float2 m = (is_r ? map_r : map_l)[j % hw];
    unsigned char* d = (is_r ? dr : dl) + j * 3;
    if (!(m.x >= -1.f && m.x <= (float)w && m.y >= -1.f && m.y <= (float)h)) { d[0] = 0; d[1] = 0; d[2] = 0; return; }
    const float fx0 = floorf(m.x), fy0 = floorf(m.y);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const float fx = m.x - fx0, fy = m.y - fy0;
    const unsigned char* s = (is_r ? right : left) + (j / hw) * hw * 3;
    const bool in_x0 = x0 >= 0 && x0 < w, in_x1 = x0 + 1 < w, in_y0 = y0 >= 0 && y0 < h, in_y1 = y0 + 1 < h;
    const unsigned char* r0 = s + (size_t)(in_y0 ? y0 : 0) * w * 3;
    const unsigned char* r1 = s + (size_t)(in_y1 ? y0 + 1 : 0) * w * 3;
    const int c0 = (in_x0 ? x0 : 0) * 3, c1 = (in_x1 ? x0 + 1 : 0) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float tl = in_y0 && in_x0 ? (float)r0[c0 + c] : 0.f, tr = in_y0 && in_x1 ? (float)r0[c1 + c] : 0.f;
        const float bl = in_y1 && in_x0 ? (float)r1[c0 + c] : 0.f, br = in_y1 && in_x1 ? (float)r1[c1 + c] : 0.f;
        const float top = tl + (tr - tl) * fx;
        const float bot = bl + (br - bl) * fx;
        d[c] = (unsigned char)min(max(__float2int_rn(top + (bot - top) * fy), 0), 255);
    }
}

int rectify_u8(const unsigned char* left, const unsigned char* right, const float* map_left, const float* map_right, int B,
               int h, int w, unsigned char* dst_left, unsigned char* dst_right, cudaStream_t st) {
    MS_REQUIRE(B >= 1 && h >= 1 && w >= 1, "rectify_u8: bad geometry");
    MS_REQUIRE(left && map_left && dst_left, "rectify_u8: null pointer");
    MS_REQUIRE(!right == !map_right && !right == !dst_right, "rectify_u8: the right frame needs its own map and output");
    MS_REQUIRE(((reinterpret_cast<uintptr_t>(map_left) | reinterpret_cast<uintptr_t>(map_right)) & 7) == 0,
               "rectify_u8: maps must be 8-byte aligned");
    const int ncam = right ? 2 : 1;
    const size_t total = (size_t)ncam * B * h * w;
    launch_k(rectify_u8_kernel, dim3((unsigned)cdivz(total, 256)), dim3(256), 0, st, left, right,
             reinterpret_cast<const float2*>(map_left), reinterpret_cast<const float2*>(map_right), ncam, B, h, w, dst_left,
             dst_right);
    return check_launch("rectify_u8");
}

}  // namespace ms
