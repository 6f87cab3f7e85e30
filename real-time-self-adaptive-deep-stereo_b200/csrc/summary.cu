// Colour maps of disparities for the TensorBoard summaries of the adaptation drivers (reference
// Stereo_Online_Adaptation.py:131-140, Stereo_Continual_Adaptation.py:135-145).  Runs once per 100 frames.
//
//   colorize             preprocessing.colorize_img (Data_utils/preprocessing.py:91-117): [B,H,W,1] -> float [B,H,W,3]
//   colorize_summary_u8  the same for image 0 only (tf.summary.image(..., max_outputs=1)), then ImageSummary's float ->
//                        uint8 normalization, so that only the H*W*3 bytes of the PNG's pixels leave the device
//
// Passes over the map: one fixed-grid min/max over the whole batch (skipped when vmin and vmax are both given) and one
// colorize pass.  The summary form needs the maximum of the gathered colours of image 0 before it can scale them, so it
// splits the colorize pass in two kernels: the second re-reads image 0 from L2, where the first has just left it.
#include <algorithm>
#include <math.h>
#include "common.cuh"

namespace ms {

constexpr int CZ_THREADS = 256;
constexpr int CZ_MAX_BLOCKS = 2 * NUM_SMS;
// workspace: value min/max partials [0, 2*CZ_MAX_BLOCKS), colour min/max partials [2*CZ_MAX_BLOCKS, 4*CZ_MAX_BLOCKS)
size_t colorize_workspace_floats() { return 4 * CZ_MAX_BLOCKS; }

// the grid depends on the element count only, so every partial slot holds the same elements on every call
static int cz_blocks(size_t n) {
    return (int)std::min<size_t>(CZ_MAX_BLOCKS, std::max<size_t>(1, cdivz(n, (size_t)CZ_THREADS * 8)));
}

// block-wide min and max (fminf / fmaxf: a NaN input is ignored); the result is returned to every thread
__device__ void cz_block_minmax(float& lo, float& hi) {
    __shared__ float slo[CZ_THREADS / 32], shi[CZ_THREADS / 32];
    for (int o = 16; o; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();                                   // the arrays may still be read by a previous call
    if (lane == 0) { slo[wid] = lo; shi[wid] = hi; }
    __syncthreads();
    lo = INFINITY; hi = -INFINITY;
    for (int i = 0; i < CZ_THREADS / 32; ++i) { lo = fminf(lo, slo[i]); hi = fmaxf(hi, shi[i]); }
}

__device__ void cz_reduce_partials(const float* part, int nparts, float& lo, float& hi) {
    lo = INFINITY; hi = -INFINITY;
    for (int i = threadIdx.x; i < nparts; i += CZ_THREADS) { lo = fminf(lo, part[2 * i]); hi = fmaxf(hi, part[2 * i + 1]); }
    cz_block_minmax(lo, hi);
}

// LUT row of a value, or row 256 (zeros) where the reference's gather index falls outside [0, 255]: TF's GPU gather writes
// zeros there.
// Same float32 operations as the reference graph, each rounded on its own (no FMA contraction):
// to_int32(round(((v - vmin) / (vmax - vmin)) * 255)), tf.round = rintf (ties to even).  vmax == vmin gives 0/0 = NaN,
// which is no index: a constant map comes out black.
__device__ __forceinline__ int cz_index(float v, float vmin, float vrange) {
    const float x = rintf(__fmul_rn(__fdiv_rn(__fsub_rn(v, vmin), vrange), 255.f));
    return (x >= 0.f && x <= 255.f) ? (int)x : 256;
}

struct CzRange { int use_vmin, use_vmax; float vmin, vmax; };

// every block: the LUT and a zero row 256 into shared memory, and (vmin, vmax - vmin) from the given values or the min/max partials
__device__ void cz_setup(const float* __restrict__ lut, const float* __restrict__ part, int nparts, CzRange r, float* s_lut,
                         float& vmin, float& vrange) {
    for (int i = threadIdx.x; i < 257 * 3; i += CZ_THREADS) s_lut[i] = i < 256 * 3 ? lut[i] : 0.f;
    float lo = 0.f, hi = 0.f;
    if (nparts > 0) cz_reduce_partials(part, nparts, lo, hi);
    vmin = r.use_vmin ? r.vmin : lo;
    const float vmax = r.use_vmax ? r.vmax : hi;
    vrange = __fsub_rn(vmax, vmin);
    __syncthreads();
}

__global__ void __launch_bounds__(CZ_THREADS) cz_minmax_kernel(const float* __restrict__ v, size_t n, float* __restrict__ part) {
    pdl_prologue();
    float lo = INFINITY, hi = -INFINITY;
    for (size_t i = (size_t)blockIdx.x * CZ_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * CZ_THREADS) {
        const float x = v[i];
        lo = fminf(lo, x); hi = fmaxf(hi, x);
    }
    cz_block_minmax(lo, hi);
    if (threadIdx.x == 0) { part[2 * blockIdx.x] = lo; part[2 * blockIdx.x + 1] = hi; }
}

__global__ void __launch_bounds__(CZ_THREADS) cz_colorize_kernel(const float* __restrict__ v, size_t n, const float* __restrict__ lut,
                                                                 const float* __restrict__ part, int nparts, CzRange r,
                                                                 float* __restrict__ out) {
    pdl_prologue();
    __shared__ float s_lut[257 * 3];
    float vmin, vrange;
    cz_setup(lut, part, nparts, r, s_lut, vmin, vrange);
    for (size_t i = (size_t)blockIdx.x * CZ_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * CZ_THREADS) {
        const int k = cz_index(v[i], vmin, vrange);
        float* o = out + 3 * i;
        o[0] = s_lut[3 * k]; o[1] = s_lut[3 * k + 1]; o[2] = s_lut[3 * k + 2];
    }
}

__device__ __forceinline__ bool cz_finite3(const float* c) { return isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2]); }

// min/max of the gathered colours of image 0 over its finite pixels (the first loop of ImageSummary's normalization)
__global__ void __launch_bounds__(CZ_THREADS) cz_color_range_kernel(const float* __restrict__ v, size_t hw, const float* __restrict__ lut,
                                                                    const float* __restrict__ part, int nparts, CzRange r,
                                                                    float* __restrict__ cpart) {
    pdl_prologue();
    __shared__ float s_lut[257 * 3];
    float vmin, vrange;
    cz_setup(lut, part, nparts, r, s_lut, vmin, vrange);
    float lo = INFINITY, hi = -INFINITY;
    for (size_t i = (size_t)blockIdx.x * CZ_THREADS + threadIdx.x; i < hw; i += (size_t)gridDim.x * CZ_THREADS) {
        const int k = cz_index(v[i], vmin, vrange);
        const float* c = s_lut + 3 * k;
        if (cz_finite3(c)) {
            lo = fminf(lo, fminf(c[0], fminf(c[1], c[2])));
            hi = fmaxf(hi, fmaxf(c[0], fmaxf(c[1], c[2])));
        }
    }
    cz_block_minmax(lo, hi);
    if (threadIdx.x == 0) { cpart[2 * blockIdx.x] = lo; cpart[2 * blockIdx.x + 1] = hi; }
}

// ImageSummary's float -> uint8 rule (TensorFlow's summary image op, restated from its documented behaviour: the C++
// kernel is not run by any test here, so this parity point is unpinned).  Over the finite pixels: if the minimum is >= 0 the
// image is scaled by 255 / max (0 when max < 1e-6), else by 127 / max(|min|, |max|) and offset by 128.  Each channel is
// c * scale rounded, plus offset rounded (no FMA), then truncated toward zero to uint8.  A pixel with a non-finite channel
// gets bad_color, red.
__global__ void __launch_bounds__(CZ_THREADS) cz_summary_u8_kernel(const float* __restrict__ v, size_t hw, const float* __restrict__ lut,
                                                                   const float* __restrict__ part, int nparts, CzRange r,
                                                                   const float* __restrict__ cpart, int ncparts,
                                                                   unsigned char* __restrict__ out) {
    pdl_prologue();
    __shared__ float s_lut[257 * 3];
    float vmin, vrange;
    cz_setup(lut, part, nparts, r, s_lut, vmin, vrange);
    float lo, hi;
    cz_reduce_partials(cpart, ncparts, lo, hi);
    float scale, offset;
    if (lo < 0.f) {
        const float m = fmaxf(fabsf(lo), fabsf(hi));
        scale = m < 1e-6f ? 0.f : __fdiv_rn(127.f, m);
        offset = 128.f;
    } else {
        scale = hi < 1e-6f ? 0.f : __fdiv_rn(255.f, hi);
        offset = 0.f;
    }
    for (size_t i = (size_t)blockIdx.x * CZ_THREADS + threadIdx.x; i < hw; i += (size_t)gridDim.x * CZ_THREADS) {
        const int k = cz_index(v[i], vmin, vrange);
        const float* c = s_lut + 3 * k;
        unsigned char* o = out + 3 * i;
        if (cz_finite3(c)) {
            for (int j = 0; j < 3; ++j) o[j] = (unsigned char)__float2int_rz(__fadd_rn(__fmul_rn(c[j], scale), offset));
        } else {
            o[0] = 255; o[1] = 0; o[2] = 0;
        }
    }
}

static int cz_check(const float* value, int B, int H, int W, const float* lut, const void* out, const float* ws, size_t ws_floats) {
    MS_REQUIRE(B >= 1 && H >= 1 && W >= 1, "colorize: bad geometry");
    MS_REQUIRE(value && lut && out, "colorize: null pointer");
    MS_REQUIRE(ws && ws_floats >= colorize_workspace_floats(), "colorize: workspace smaller than ms_colorize_workspace_floats()");
    return 0;
}

// the batch-wide min/max partials, or none when both ends of the range are given
static int cz_minmax(const float* value, size_t n, CzRange r, float* ws, int& nparts, cudaStream_t st) {
    nparts = 0;
    if (r.use_vmin && r.use_vmax) return 0;
    nparts = cz_blocks(n);
    launch_k(cz_minmax_kernel, dim3(nparts), dim3(CZ_THREADS), 0, st, value, n, ws);
    return check_launch("colorize min/max");
}

int colorize(const float* value, int B, int H, int W, const float* lut, int use_vmin, float vmin, int use_vmax, float vmax,
             float* out, float* ws, size_t ws_floats, cudaStream_t st) {
    const CzRange r{use_vmin, use_vmax, vmin, vmax};
    if (int rc = cz_check(value, B, H, W, lut, out, ws, ws_floats)) return rc;
    const size_t n = (size_t)B * H * W;
    int nparts;
    if (int rc = cz_minmax(value, n, r, ws, nparts, st)) return rc;
    launch_k(cz_colorize_kernel, dim3(cz_blocks(n)), dim3(CZ_THREADS), 0, st, value, n, lut, (const float*)ws, nparts, r, out);
    return check_launch("colorize");
}

int colorize_summary_u8(const float* value, int B, int H, int W, const float* lut, int use_vmin, float vmin, int use_vmax,
                        float vmax, unsigned char* out, float* ws, size_t ws_floats, cudaStream_t st) {
    const CzRange r{use_vmin, use_vmax, vmin, vmax};
    if (int rc = cz_check(value, B, H, W, lut, out, ws, ws_floats)) return rc;
    int nparts;
    if (int rc = cz_minmax(value, (size_t)B * H * W, r, ws, nparts, st)) return rc;
    const size_t hw = (size_t)H * W;
    const int g = cz_blocks(hw);
    float* cpart = ws + 2 * CZ_MAX_BLOCKS;
    launch_k(cz_color_range_kernel, dim3(g), dim3(CZ_THREADS), 0, st, value, hw, lut, (const float*)ws, nparts, r, cpart);
    launch_k(cz_summary_u8_kernel, dim3(g), dim3(CZ_THREADS), 0, st, value, hw, lut, (const float*)ws, nparts, r,
             (const float*)cpart, g, out);
    return check_launch("colorize summary image", 2);
}

}  // namespace ms
