// Resampling / elementwise kernels of the hot path (all HBM-bound, one pass each).
//
//   pad_reflect          preprocessing.pad_image                 (reference Data_utils/preprocessing.py:7-29)
//   resize_bilinear      tf.image.resize_images legacy bilinear  (Nets/MadNet.py:69,274,293,312,331,362;
//                        + resize_image_with_crop_or_pad centre crop, MadNet.py:70,363) with the
//                        relu / x20 / x(-20) scalings of MadNet._make_disp fused in
//   resize_bilinear_bwd  its transpose (what tf.gradients builds), separable two-pass gather => deterministic
//   leaky_bwd            gradient of tf.maximum(alpha*x, x)      (Nets/MadNet.py:366-367)
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
__device__ __forceinline__ Lerp lerp_coeff(int o, float scale, int in_size) {
    // TF 1.x legacy bilinear: src = dst*scale, no half-pixel centres
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

}  // namespace ms
