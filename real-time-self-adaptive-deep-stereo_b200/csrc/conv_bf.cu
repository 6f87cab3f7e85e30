// conv_bf: wgmma implicit-GEMM convolution on split 16-bit operands -- the default tensor-core path of the conv stacks.
//
// Replaces the cuDNN calls behind tf.nn.conv2d / tf.nn.atrous_conv2d (reference Nets/sharedLayers.py:58,72) and their
// input gradients for the estimator / context / pyramid layers of MADNet (Nets/MadNet.py:73-171,173-249) and the
// DispNet encoder / refinement convs (Nets/DispNet.py:77-140).
//
//   * operands are PRE-SPLIT: every tensor that feeds a convolution also exists as two 16-bit planes (x ~= hi + lo),
//     written by the producing kernel's epilogue; weights are split once per update.  The main loop is the canonical
//     TMA -> wgmma -> epilogue pipeline, no splitter.
//       forward operands : fp16 planes of x/16 and of w  (hi = fp16, lo = fp16 of the remainder: 22 mantissa bits,
//                          ~2^-22 relative product error -- fp32-grade, so no extra relu / floor / |.| kink flips; the
//                          1/16 pre-scale keeps |x| <= 1e6 inside the fp16 range, undone exactly in the epilogue)
//       gradient operands: bf16 planes (hi + lo: 16 mantissa bits, ~2^-16, full fp32 exponent range for 1e-9 gradients)
//   * three 16-bit MMAs per K step (w_lo*x_hi + w_hi*x_lo into one accumulator, w_hi*x_hi into another) at the
//     bf16/fp16 tensor rate (twice the tf32 rate).
//   * the GEMM is transposed ("swap AB"): M = output channels (128 per CTA: two warpgroups of m64 wgmma), N = up to 128
//     output pixels per CTA.  One weight tile serves all N pixels, and the epilogue maps consecutive threads to
//     consecutive channels of one pixel, so every NHWC store is a coalesced line.
//   * K blocks of 64 channels (128-byte rows, SWIZZLE_128B) whenever cin > 32, else 32 (64-byte rows, SWIZZLE_64B).
//   * weights are stored PRE-TILED in their shared-memory image (per (M block, tap, K block): hi tile | lo tile,
//     swizzle applied by the prep kernel) and arrive as ONE 1-D bulk copy per tap instead of 2 x 128 TMA rows.
//   * A tile's pixels are `TW` wide and N/TW high.  For each filter column the kernel loads ONE halo patch
//     (N/TW + (kh-1)*dilation rows) per K block; the kh taps of that column are row offsets into the patch
//     (patch rows are whole swizzle atoms, so a tap is just a different descriptor start address).
//     Stride-2 convolutions use TMA element strides {1,2,2,1}: a patch then holds every second pixel / row.
//   * split-K over (K block, patch) units for small maps; the last-arriving CTA of a tile reduces the partial
//     sums in fixed order (deterministic) and runs the epilogue -- no separate reduce launch.
//
// Warpgroup roles (384 threads): warpgroup 0 = TMA producer (one warp issues), warpgroups 1-2 = wgmma on output channels
// [0, 64) / [64, 128) of the M block, then the epilogue.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace ms {

constexpr int BF_THREADS = 384;
constexpr int BF_MAX_N = 128;        // pixels per CTA: two fp32 accumulators of N/2 registers per thread
constexpr int BF_MAX_PATCH = 16;
constexpr int BF_MAX_TAPS = 49;
constexpr int BF_STAGE_LD = 132;     // floats per pixel row of the epilogue staging tile (128 channels + 4: no bank conflicts)

struct BfPatch { short dx, dy, ntaps, tap0; };
struct BfTap { short row_off, widx; };

struct ConvBfParams {
    int H, W, NB;                 // output lattice handled by this launch (tile validity)
    int Hout, Wout, os, oy0, ox0; // output tensor; lattice point (j) is output pixel j * os + o0
    int TW, tw_shift, N;          // pixel tile: TW wide (power of two), N pixels
    int tiles_x, tiles_y;
    int sx;                       // input coordinate = out * sx + patch.d
    int kblocks, n_patches;
    int kch;                      // channels per K block: 32 (64-byte rows, SWIZZLE_64B) or 64 (128-byte rows, SWIZZLE_128B)
    int taps_total;
    uint32_t slot_bytes;          // bytes of one patch plane in shared memory
    uint32_t wtile_bytes;         // bytes of one weight tile plane (128 rows x kch x 2)
    int NP, NW;
    int fmt;                      // operand format: 0 = bf16 planes, 1 = fp16 planes (activation planes hold x * scale)
    float acc_scale;              // multiplies the accumulator (1 / scale of the input planes, a power of two: exact)
    int cout;
    int ksplit;
    const unsigned char* wtiles;  // pre-tiled weights [M block][tap][K block][hi tile | lo tile]
    float* part; unsigned int* tickets;
    float* y; int ycs;
    const float* bias; float alpha;
    const float* res; int res_cs;
    const float* mask; int mask_cs; float mask_alpha;
    int accumulate;
    void* ohi; void* olo; int ocs; int ofmt; float oscale;   // optional output planes (format, stored value = t * oscale)
    BfPatch patch[BF_MAX_PATCH];
    BfTap tap[BF_MAX_TAPS];
};

__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(s_addr(dst)), "l"(src), "r"(bytes), "r"(s_addr(bar)) : "memory");
}

// 16-bit split of a float: fmt 0 -> bf16 hi/lo of v (any magnitude), fmt 1 -> fp16 hi/lo of v * scale (22 mantissa bits while
// |v * scale| stays inside fp16's normal range; saturating, so an out-of-range value degrades instead of becoming inf)
__device__ __forceinline__ void split16(float v, int fmt, float scale, unsigned short& hi, unsigned short& lo) {
    if (fmt == 0) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        const __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
        hi = __bfloat16_as_ushort(h); lo = __bfloat16_as_ushort(l);
    } else {
        const float s = v * scale;
        asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(hi) : "f"(s));
        const float r = s - __half2float(__ushort_as_half(hi));
        asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(lo) : "f"(r));
    }
}

// N: pixels per CTA (64, 96 or 128); BF: 1 = bf16 operand planes, 0 = fp16
template <int N, int BF>
__global__ void __launch_bounds__(BF_THREADS, 1)
conv_bf_kernel(const __grid_constant__ CUtensorMap mapXh, const __grid_constant__ CUtensorMap mapXl,
               const __grid_constant__ ConvBfParams p) {
    extern __shared__ unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t pfull[4], pempty[4], wfull[8], wempty[8];
    __shared__ int last_flag;

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const uint32_t base = (s_addr(smem_dyn) + 1023u) & ~1023u;
    unsigned char* gbase = smem_dyn + (base - s_addr(smem_dyn));
    const uint32_t pslot = 2u * p.slot_bytes;                 // hi plane | lo plane
    const uint32_t w_off = (uint32_t)p.NP * pslot;
    const uint32_t wslot = 2u * p.wtile_bytes;                // hi tile | lo tile

    int bid = blockIdx.x;
    const int tx = bid % p.tiles_x; bid /= p.tiles_x;
    const int ty = bid % p.tiles_y;
    const int img = bid / p.tiles_y;
    const int TH = N >> p.tw_shift;
    const int x0 = tx * p.TW, y0 = ty * TH;
    const int units = p.kblocks * p.n_patches;
    const int u0 = (int)(((long)blockIdx.z * units) / p.ksplit), u1 = (int)(((long)(blockIdx.z + 1) * units) / p.ksplit);
    // programmatic dependent launch (common.cuh): the next kernel's CTAs may become resident as soon as every CTA of this
    // grid has started; this kernel's own global traffic starts only after pdl_wait() below
    pdl_trigger();

    if (threadIdx.x == 0) {
        // full: one arrival (the producer's expect_tx) + the bytes; empty: one arrival per MMA warp (8)
        for (int i = 0; i < p.NP; ++i) { mb_init(&pfull[i], 1); mb_init(&pempty[i], 8); }
        for (int i = 0; i < p.NW; ++i) { mb_init(&wfull[i], 1); mb_init(&wempty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_wait();                                               // the barrier set-up above overlapped the previous kernel's tail

    if (warp < 4) {
        // ================= producer: halo patches by TMA (per K block x filter column) + weight tiles by bulk copy (per tap) ===
        if (warp == 0) {
            const bool leader = elect_one();               // warp-uniform loop, elected lane issues (tc_ptx.cuh:elect_one)
            int ps = 0, ws = 0;
            uint32_t pph = 0, wph = 0;
            const unsigned char* wbase = p.wtiles + (size_t)blockIdx.y * p.taps_total * p.kblocks * wslot;
            int kb = u0 / p.n_patches, pi = u0 - kb * p.n_patches;
            for (int u = u0; u < u1; ++u) {
                const BfPatch pt = p.patch[pi];
                mb_wait(&pempty[ps], pph ^ 1u);
                unsigned char* dst = gbase + (size_t)ps * pslot;
                if (leader) {
                    mb_expect_tx(&pfull[ps], pslot);
                    tma_load_4d(dst, &mapXh, &pfull[ps], kb * p.kch, x0 * p.sx + pt.dx, y0 * p.sx + pt.dy, img);
                    tma_load_4d(dst + p.slot_bytes, &mapXl, &pfull[ps], kb * p.kch, x0 * p.sx + pt.dx, y0 * p.sx + pt.dy, img);
                }
                if (++ps == p.NP) { ps = 0; pph ^= 1u; }
                for (int t = pt.tap0; t < pt.tap0 + pt.ntaps; ++t) {
                    mb_wait(&wempty[ws], wph ^ 1u);
                    if (leader) {
                        mb_expect_tx(&wfull[ws], wslot);
                        bulk_load(gbase + w_off + (size_t)ws * wslot, wbase + ((size_t)p.tap[t].widx * p.kblocks + kb) * wslot, wslot, &wfull[ws]);
                    }
                    if (++ws == p.NW) { ws = 0; wph ^= 1u; }
                }
                if (++pi == p.n_patches) { pi = 0; ++kb; }
            }
        }
        return;
    }

    // ================= MMA warpgroups: channels [64 * mg, 64 * mg + 64) of the M block, all N pixels =================
    const int mg = (warp >> 2) - 1;
    const int ct = threadIdx.x - 128;                         // 0..255 over both MMA warpgroups
    float acc_x[N / 2], acc_m[N / 2];                         // cross terms (w_lo*x_hi + w_hi*x_lo) and w_hi*x_hi
#pragma unroll
    for (int i = 0; i < N / 2; ++i) { acc_x[i] = 0.f; acc_m[i] = 0.f; }
    {
        const bool sw128 = p.kch == 64;
        const uint32_t row_unit = (uint32_t)p.kch * 2u;       // bytes of one K-major row (one pixel / one channel)
        const uint32_t sbo = sw128 ? 1024u : 512u;
        const int k16 = p.kch >> 4;
        const uint32_t row_bytes = (uint32_t)p.TW * row_unit;
        int ps = 0, ws = 0;
        uint32_t pph = 0, wph = 0;
        int pend_w = -1, pend_p = -1;                         // ring slots read by the MMAs still in flight
        int pi = u0 % p.n_patches;
        for (int u = u0; u < u1; ++u) {
            const BfPatch pt = p.patch[pi];
            mb_wait(&pfull[ps], pph);
            const uint32_t pb = base + (uint32_t)ps * pslot;
            for (int t = pt.tap0; t < pt.tap0 + pt.ntaps; ++t) {
                mb_wait(&wfull[ws], wph);
                const uint32_t boff = (uint32_t)p.tap[t].row_off * row_bytes;
                const uint64_t xh = wg_desc(pb + boff, 16u, sbo, sw128), xl = wg_desc(pb + p.slot_bytes + boff, 16u, sbo, sw128);
                const uint32_t wb = base + w_off + (uint32_t)ws * wslot + (uint32_t)mg * 64u * row_unit;
                const uint64_t wh = wg_desc(wb, 16u, sbo, sw128), wl = wg_desc(wb + p.wtile_bytes, 16u, sbo, sw128);
                wg_fence_acc(acc_x); wg_fence_acc(acc_m);
                wg_fence();
                for (int j = 0; j < k16; ++j) {                // K = 16 elements = 32 bytes inside the swizzle row
                    const uint64_t o = (uint64_t)(j * 2);
                    Wgmma<N, BF, 0, 0>::mma(acc_x, wl + o, xh + o);
                    Wgmma<N, BF, 0, 0>::mma(acc_x, wh + o, xl + o);
                    Wgmma<N, BF, 0, 0>::mma(acc_m, wh + o, xh + o);
                }
                wg_commit();
                wg_wait<1>();                                 // the previous tap's MMAs are done with their operands
                wg_fence_acc(acc_x); wg_fence_acc(acc_m);
                if (lane == 0) {
                    if (pend_w >= 0) mb_arrive(&wempty[pend_w]);
                    if (pend_p >= 0) mb_arrive(&pempty[pend_p]);
                }
                pend_w = ws;
                pend_p = (t == pt.tap0 + pt.ntaps - 1) ? ps : -1;
                if (++ws == p.NW) { ws = 0; wph ^= 1u; }
            }
            if (++ps == p.NP) { ps = 0; pph ^= 1u; }
            if (++pi == p.n_patches) pi = 0;
        }
        wg_wait<0>();
        wg_fence_acc(acc_x); wg_fence_acc(acc_m);
    }

    // ================= epilogue: accumulators -> staging tile [pixel][channel] in the (now idle) pipeline buffers ==========
    float* const stage = reinterpret_cast<float*>(gbase);
    named_sync(1, 256);                                       // both warpgroups' MMAs have finished reading the rings
    {
        const int row = mg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int col = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            float* s0 = stage + (size_t)(8 * j + col) * BF_STAGE_LD + row;
            s0[0] = acc_x[4 * j] + acc_m[4 * j];
            s0[BF_STAGE_LD] = acc_x[4 * j + 1] + acc_m[4 * j + 1];
            s0[8] = acc_x[4 * j + 2] + acc_m[4 * j + 2];
            s0[BF_STAGE_LD + 8] = acc_x[4 * j + 3] + acc_m[4 * j + 3];
        }
    }
    named_sync(1, 256);

    // thread <-> 4 consecutive channels of one pixel: 128-bit loads / stores for y, residual, mask and accumulate, 64-bit
    // stores for the two 16-bit planes
    const int chb = blockIdx.y * 128;
    const int cpp = min(32, (p.cout - chb + 3) >> 2);         // 4-channel chunks per pixel in this M block
    const int twm = p.TW - 1;
    const size_t img_pix = (size_t)img * p.Hout;
    const float acc_scale = p.acc_scale, alpha = p.alpha;
    const bool has_res = p.res != nullptr, has_mask = p.mask != nullptr, has_acc = p.accumulate != 0, has_pl = p.ohi != nullptr;
    unsigned short* const ohi = reinterpret_cast<unsigned short*>(p.ohi);
    unsigned short* const olo = reinterpret_cast<unsigned short*>(p.olo);
    const bool vec_ok = (p.cout & 3) == 0 && (p.ycs & 3) == 0 && (reinterpret_cast<uintptr_t>(p.y) & 15) == 0 &&
                        (!has_res || ((p.res_cs & 3) == 0 && (reinterpret_cast<uintptr_t>(p.res) & 15) == 0)) &&
                        (!has_mask || ((p.mask_cs & 3) == 0 && (reinterpret_cast<uintptr_t>(p.mask) & 15) == 0)) &&
                        (!has_pl || ((p.ocs & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.ohi) | reinterpret_cast<uintptr_t>(p.olo)) & 7) == 0));
    auto finish4 = [&](int col, int c4, float (&v)[4]) {
        const int yy = y0 + (col >> p.tw_shift), xx = x0 + (col & twm);
        if (yy >= p.H || xx >= p.W) return;
        const int ch = chb + c4 * 4;
        const size_t pix = (img_pix + (size_t)(yy * p.os + p.oy0)) * p.Wout + (size_t)(xx * p.os + p.ox0);
        if (vec_ok) {
            float4 t = make_float4(v[0] * acc_scale, v[1] * acc_scale, v[2] * acc_scale, v[3] * acc_scale);
            if (p.bias) { const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + ch)); t.x += b.x; t.y += b.y; t.z += b.z; t.w += b.w; }
            t.x = fmaxf(alpha * t.x, t.x); t.y = fmaxf(alpha * t.y, t.y); t.z = fmaxf(alpha * t.z, t.z); t.w = fmaxf(alpha * t.w, t.w);
            if (has_res) { const float4 r = *reinterpret_cast<const float4*>(p.res + pix * p.res_cs + ch); t.x += r.x; t.y += r.y; t.z += r.z; t.w += r.w; }
            float4* yp = reinterpret_cast<float4*>(p.y + pix * p.ycs + ch);
            if (has_acc) { const float4 o = *yp; t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w; }
            if (has_mask) {
                const float4 m = *reinterpret_cast<const float4*>(p.mask + pix * p.mask_cs + ch);
                t.x *= m.x > 0.f ? 1.f : p.mask_alpha; t.y *= m.y > 0.f ? 1.f : p.mask_alpha;
                t.z *= m.z > 0.f ? 1.f : p.mask_alpha; t.w *= m.w > 0.f ? 1.f : p.mask_alpha;
            }
            *yp = t;
            if (has_pl) {
                unsigned short h[4], l[4];
                split16(t.x, p.ofmt, p.oscale, h[0], l[0]); split16(t.y, p.ofmt, p.oscale, h[1], l[1]);
                split16(t.z, p.ofmt, p.oscale, h[2], l[2]); split16(t.w, p.ofmt, p.oscale, h[3], l[3]);
                uint2 hv, lv;
                hv.x = (uint32_t)h[0] | ((uint32_t)h[1] << 16); hv.y = (uint32_t)h[2] | ((uint32_t)h[3] << 16);
                lv.x = (uint32_t)l[0] | ((uint32_t)l[1] << 16); lv.y = (uint32_t)l[2] | ((uint32_t)l[3] << 16);
                *reinterpret_cast<uint2*>(ohi + pix * p.ocs + ch) = hv;
                *reinterpret_cast<uint2*>(olo + pix * p.ocs + ch) = lv;
            }
            return;
        }
        // scalar path (channel counts / strides that are not multiples of 4)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (ch + j >= p.cout) break;
            float t = v[j] * acc_scale + (p.bias ? __ldg(p.bias + ch + j) : 0.f);
            t = fmaxf(alpha * t, t);
            if (has_res) t += p.res[pix * p.res_cs + ch + j];
            if (has_acc) t += p.y[pix * p.ycs + ch + j];
            if (has_mask) t *= (p.mask[pix * p.mask_cs + ch + j] > 0.f) ? 1.f : p.mask_alpha;
            p.y[pix * p.ycs + ch + j] = t;
            if (has_pl) {
                unsigned short h, l;
                split16(t, p.ofmt, p.oscale, h, l);
                ohi[pix * p.ocs + ch + j] = h;
                olo[pix * p.ocs + ch + j] = l;
            }
        }
    };

    const int items = N * cpp;
    if (p.ksplit == 1) {
        for (int i = ct; i < items; i += 256) {
            const int col = i / cpp, c4 = i - col * cpp;
            const float4 s = *reinterpret_cast<const float4*>(stage + (size_t)col * BF_STAGE_LD + c4 * 4);
            float v[4] = {s.x, s.y, s.z, s.w};
            finish4(col, c4, v);
        }
        return;
    }
    // raw partial sums: part[(z * n_tiles + tile) * N + col][128 channels]
    const int tile_lin = blockIdx.x * gridDim.y + blockIdx.y;
    const size_t n_tiles = (size_t)gridDim.x * gridDim.y;
    {
        float* mine = p.part + ((size_t)blockIdx.z * n_tiles + tile_lin) * N * 128;
        for (int i = ct; i < N * 32; i += 256) {
            const int col = i >> 5, c4 = i & 31;
            *reinterpret_cast<float4*>(mine + (size_t)col * 128 + c4 * 4) =
                *reinterpret_cast<const float4*>(stage + (size_t)col * BF_STAGE_LD + c4 * 4);
        }
    }
    __threadfence();
    named_sync(1, 256);
    if (ct == 0) {
        const unsigned int old = atomicAdd(p.tickets + tile_lin, 1u);
        const int last = (old == (unsigned int)(p.ksplit - 1)) ? 1 : 0;
        if (last) p.tickets[tile_lin] = 0u;        // self-resetting for the next launch
        last_flag = last;
    }
    named_sync(1, 256);
    if (!last_flag) return;
    __threadfence();
    const float* col0 = p.part + (size_t)tile_lin * N * 128;
    const size_t zstride = n_tiles * (size_t)N * 128;
    for (int i = ct; i < items; i += 256) {
        const int col = i / cpp, c4 = i - col * cpp;
        const float* src = col0 + (size_t)col * 128 + c4 * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (int z = 0; z < p.ksplit; ++z) {                  // fixed order: deterministic
            const float4 a = __ldcg(reinterpret_cast<const float4*>(src + (size_t)z * zstride));
            v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w;
        }
        finish4(col, c4, v);
    }
}

// ------------------------------------------------------------------------------------------------
// 16-bit planes of an fp32 NHWC view (producers that are not conv_bf epilogues: correlation, resize, loss seeds ...)
// ------------------------------------------------------------------------------------------------
__global__ void split_planes_kernel(const float* __restrict__ x, int xcs, int C, size_t pixels,
                                    unsigned short* __restrict__ hi, unsigned short* __restrict__ lo, int pcs, int fmt, float scale) {
    pdl_prologue();
    const int cq = (C + 3) >> 2;
    const size_t total = pixels * cq;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / cq;
        const int c = (int)(i - pix * cq) * 4;
        const float* src = x + pix * xcs + c;
        unsigned short h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float v = (c + j < C) ? src[j] : 0.f;
            split16(v, fmt, scale, h[j], l[j]);
        }
        unsigned short* dh = hi + pix * pcs + c;
        unsigned short* dl = lo + pix * pcs + c;
        if (c + 4 <= pcs) {
            *reinterpret_cast<uint2*>(dh) = *reinterpret_cast<const uint2*>(h);
            *reinterpret_cast<uint2*>(dl) = *reinterpret_cast<const uint2*>(l);
        } else {
            for (int j = 0; j < 4 && c + j < pcs; ++j) { dh[j] = h[j]; dl[j] = l[j]; }
        }
    }
}

int split_planes(const TView& x, const ActPlanes& pl, cudaStream_t st) {
    MS_REQUIRE(pl.hi && pl.lo && pl.cs >= x.c && (pl.cs & 7) == 0, "split_planes: bad plane buffers");
    const size_t total = x.pixels() * ((x.c + 3) / 4);
    const unsigned grid = (unsigned)std::min<size_t>(cdivz(total, 256), NUM_SMS * 16);
    launch_k(split_planes_kernel, dim3(grid), dim3(256), 0, st, x.p, x.cs, x.c, x.pixels(), reinterpret_cast<unsigned short*>(pl.hi),
                                              reinterpret_cast<unsigned short*>(pl.lo), pl.cs, pl.fmt, pl.fmt == 1 ? pl.scale : 1.f);
    return check_launch("split_planes");
}

// ------------------------------------------------------------------------------------------------
// weight preparation: the shared-memory image of every (M block, tap, K block) tile, hi tile | lo tile, swizzled,
// from canonical fp32 HWIO, batched over layers
//   transposed_src = 1 : src is [tap][K][M]  (forward conv: K = cin, M = cout)
//   transposed_src = 0 : src is [tap][M][K]  (dgrad: M = cin, K = cout)
// ------------------------------------------------------------------------------------------------
__global__ void bf_prep_weights_kernel(const BfPrepJob* __restrict__ jobs) {
    pdl_prologue();
    const BfPrepJob j = jobs[blockIdx.y];
    const int kch = j.Kpad > 32 ? 64 : 32;
    const int kblocks = j.Kpad / kch, mblocks = j.Mpad / 128;
    const size_t tile = (size_t)128 * kch;                         // elements per tile plane
    const size_t total = (size_t)mblocks * j.taps * kblocks * tile;
    unsigned short* dst = reinterpret_cast<unsigned short*>(j.tiles);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int kk = (int)(i % kch);
        size_t q = i / kch;
        const int r = (int)(q % 128); q /= 128;
        const int kb = (int)(q % kblocks); q /= kblocks;
        const int t = (int)(q % j.taps);
        const int mb = (int)(q / j.taps);
        const int m = mb * 128 + r, k = kb * kch + kk;
        float v = 0.f;
        if (m < j.M && k < j.K)
            v = j.transposed_src ? j.src[((size_t)t * j.K + k) * j.M + m] : j.src[((size_t)t * j.M + m) * j.K + k];
        unsigned short h, l;
        if (j.fmt == 0) {
            const __nv_bfloat16 hb = __float2bfloat16_rn(v);
            h = __bfloat16_as_ushort(hb); l = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(hb)));
        } else {                                                  // weights are not pre-scaled
            const __half hh = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
            h = __half_as_ushort(hh); l = __half_as_ushort(__float2half_rn(v - __half2float(hh)));
        }
        // swizzled position inside the tile image (K-major rows of kch*2 bytes, 16-byte chunks XOR-ed with the row bits)
        const int chunk = kk >> 3, e = kk & 7;
        const int sw = kch == 64 ? (chunk ^ (r & 7)) : (chunk ^ ((r >> 1) & 3));
        const size_t off = (size_t)r * kch + (size_t)sw * 8 + e;
        const size_t tbase = ((((size_t)mb * j.taps + t) * kblocks + kb) * 2) * tile;
        dst[tbase + off] = h;
        dst[tbase + tile + off] = l;
    }
}

int bf_prep_weights(const BfPrepJob* jobs_dev, int njobs, size_t max_total, cudaStream_t st) {
    if (njobs <= 0) return 0;
    const unsigned gx = (unsigned)std::min<size_t>(cdivz(max_total / 2, 256), 512);
    launch_k(bf_prep_weights_kernel, dim3(dim3(gx, njobs)), dim3(256), 0, st, jobs_dev);
    return check_launch("bf_prep_weights");
}

void conv_bf_weight_dims(int M, int K, int& Mpad, int& Kpad) {
    Mpad = (M + 127) / 128 * 128;
    Kpad = K > 32 ? (K + 63) / 64 * 64 : 32;
}
size_t conv_bf_weight_halfs(int taps, int M, int K) {       // 16-bit elements of the tiled image, both planes
    int Mpad, Kpad; conv_bf_weight_dims(M, K, Mpad, Kpad);
    return (size_t)2 * taps * Mpad * Kpad;
}

// ------------------------------------------------------------------------------------------------
// tensor maps (16-bit planes: SWIZZLE_64B / 128B, optional element strides; fp32: SWIZZLE_128B or none), zero OOB fill, cached
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn bf_get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* q = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(q);
    }
    return fn;
}
struct BfMapKey {
    uintptr_t addr; int rank; int swz; int f32; uint64_t d[4]; uint64_t s[3]; uint32_t b[4]; uint32_t es[4];
    bool operator<(const BfMapKey& o) const { return memcmp(this, &o, sizeof(BfMapKey)) < 0; }
};
// (BFLOAT16 as the element type for fp16 planes too: TMA moves 2-byte elements, the zero fill is format-agnostic)
// swizzle_bytes: 0, 64 or 128
static int get_map(const CUtensorMap** out, bool f32, void* addr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                   const cuuint32_t* box, const cuuint32_t* estr, int swizzle_bytes) {
    static std::map<BfMapKey, CUtensorMap> cache;
    BfMapKey k;
    memset(&k, 0, sizeof k);
    k.addr = reinterpret_cast<uintptr_t>(addr); k.rank = rank; k.swz = swizzle_bytes; k.f32 = f32 ? 1 : 0;
    for (int i = 0; i < rank; ++i) { k.d[i] = dims[i]; k.b[i] = box[i]; k.es[i] = estr[i]; }
    for (int i = 0; i + 1 < rank; ++i) k.s[i] = strides_bytes[i];
    auto it = cache.find(k);
    if (it == cache.end()) {
        EncodeTiledFn enc = bf_get_encode();
        MS_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point not available");
        CUtensorMap m;
        const CUtensorMapSwizzle swz = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                       : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE);
        CUresult r = enc(&m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, addr, dims,
                         strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r)); return -1; }
        if (cache.size() >= 8192) {
            static thread_local CUtensorMap spill[16];
            static thread_local unsigned spill_i = 0;
            CUtensorMap* slot = &spill[spill_i++ & 15u];
            *slot = m;
            *out = slot;
            return 0;
        }
        it = cache.emplace(k, m).first;
    }
    *out = &it->second;
    return 0;
}
int bf_get_map(const CUtensorMap** out, void* addr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, const cuuint32_t* estr, int swizzle_bytes) {
    return get_map(out, false, addr, rank, dims, strides_bytes, box, estr, swizzle_bytes);
}
int tc_get_map(const CUtensorMap** out, void* addr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, bool swizzle128) {
    const cuuint32_t es[4] = {1, 1, 1, 1};
    return get_map(out, true, addr, rank, dims, strides_bytes, box, es, swizzle128 ? 128 : 0);
}

// ------------------------------------------------------------------------------------------------
bool conv_bf_supported(const ConvGemm& g) {
    if (g.div != 1 && !(g.div == 2 && g.mul == 1)) return false;       // forward (stride 1/2), dgrad / transposed (stride 1/2)
    if (g.mul != 1 && g.mul != 2) return false;
    if (g.mul == 2 && g.step != 1) return false;
    if (g.div == 2 && std::abs(g.step) != 1) return false;
    if (g.x.c < 3 || g.y.c < 8) return false;          // (3-channel images: the planes are padded to 8 channels, TMA zero-fills the K block)
    if (g.kh * g.kw > BF_MAX_TAPS) return false;
    if (g.y.h * g.y.w < 32) return false;
    return true;
}

int conv_bf_init() {
    static bool done = false;
    if (done) return 0;
    MS_CHECK_CUDA(cudaFuncSetAttribute(conv_bf_kernel<64, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    MS_CHECK_CUDA(cudaFuncSetAttribute(conv_bf_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    MS_CHECK_CUDA(cudaFuncSetAttribute(conv_bf_kernel<96, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    MS_CHECK_CUDA(cudaFuncSetAttribute(conv_bf_kernel<96, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    MS_CHECK_CUDA(cudaFuncSetAttribute(conv_bf_kernel<128, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    MS_CHECK_CUDA(cudaFuncSetAttribute(conv_bf_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    done = true;
    return 0;
}

size_t conv_bf_part_floats() { return (size_t)8 << 20; }    // 32 MB of split-K partial sums
size_t conv_bf_ticket_words() { return 4096; }

struct BfTapSpec { int dy, dx, widx; };     // input pixel = out_lattice * sx + (dy, dx); weight tap index

// One launch: output lattice [Hj x Wj] (output pixel = j * os + o0), gather taps `taps`, input lattice stride sx.
static int conv_bf_launch(const ConvGemm& g, const ActPlanes& xp, const void* wtiles, const ActPlanes* yp,
                          float* part, unsigned int* tickets, int Hj, int Wj, int os, int oy0, int ox0, int sx,
                          const BfTapSpec* taps, int ntaps, int taps_total, cudaStream_t st) {
    const int K = g.x.c, M = g.y.c;
    int Mpad, Kpad; conv_bf_weight_dims(M, K, Mpad, Kpad);
    static ConvBfParams p;          // large (tables): filled in place, passed by value to the launch
    memset(&p, 0, sizeof p);
    p.H = Hj; p.W = Wj; p.NB = g.y.n; p.sx = sx;
    p.Hout = g.y.h; p.Wout = g.y.w; p.os = os; p.oy0 = oy0; p.ox0 = ox0;
    p.kch = Kpad > 32 ? 64 : 32;
    p.kblocks = Kpad / p.kch; p.cout = M; p.taps_total = taps_total;
    p.wtile_bytes = 128u * (uint32_t)p.kch * 2u;
    p.fmt = xp.fmt; p.acc_scale = xp.fmt == 1 ? 1.f / xp.scale : 1.f;
    MS_REQUIRE(xp.fmt == 0 || xp.scale > 0.f, "conv_bf: fp16 planes need a positive scale");
    const uint32_t row_unit = (uint32_t)p.kch * 2u;                 // bytes of one pixel of a patch plane
    // ---- patches: taps of one filter column (same dx; same row parity for an input lattice of stride 2) share a halo
    //      patch; a tap is a row offset into it
    auto posmod = [](int a, int m) { return ((a % m) + m) % m; };
    bool used[BF_MAX_TAPS] = {false};
    int np = 0, nt = 0, max_off = 0;
    for (int i = 0; i < ntaps; ++i) {
        if (used[i]) continue;
        int first_dy = taps[i].dy;
        for (int j = i; j < ntaps; ++j)
            if (!used[j] && taps[j].dx == taps[i].dx && posmod(taps[j].dy - taps[i].dy, sx) == 0) first_dy = std::min(first_dy, taps[j].dy);
        MS_REQUIRE(np < BF_MAX_PATCH, "conv_bf: too many patches");
        BfPatch& pt = p.patch[np];
        pt.dx = (short)taps[i].dx; pt.dy = (short)first_dy; pt.tap0 = (short)nt; pt.ntaps = 0;
        for (int j = i; j < ntaps; ++j) {
            if (used[j] || taps[j].dx != taps[i].dx || posmod(taps[j].dy - taps[i].dy, sx) != 0) continue;
            used[j] = true;
            const int off = (taps[j].dy - first_dy) / sx;
            p.tap[nt].row_off = (short)off; p.tap[nt].widx = (short)taps[j].widx;
            max_off = std::max(max_off, off);
            ++nt; ++pt.ntaps;
        }
        ++np;
    }
    // ---- pixel tile TW x TH (N = TW * TH MMA columns, a multiple of 32, 64 <= N <= BF_MAX_N).  The tile shape decides
    //      how many of the SMs work in the last wave: cost = waves x (N + fixed overhead in pixel units); ties go to the
    //      taller tile (smaller halo).
    const int mblocks = Mpad / 128;
    int N = 64, TW = 8;
    long best = -1; int best_th = 0;
    const int tws[3] = {8, 16, 32};
    for (int wi = 0; wi < 3; ++wi) {
        const int tw = tws[wi];
        if (tw * sx > 256) continue;
        for (int th = 1; th * tw <= BF_MAX_N; ++th) {
            const int n = th * tw;
            if (n < 64 || (n & 31)) continue;
            if ((th + max_off) * sx > 256) continue;
            const long tiles = (long)g.y.n * cdiv(Wj, tw) * cdiv(Hj, th) * mblocks;
            // (halo rows are loaded, not multiplied: a quarter weight keeps 32 x 2 tiles for the cases that save a wave)
            const long cost = cdiv((int)std::min<long>(tiles, 1 << 30), NUM_SMS) * (long)(n + 32 + max_off * tw / 4);
            if (best < 0 || cost < best || (cost == best && th > best_th)) { best = cost; best_th = th; N = n; TW = tw; }
        }
    }
    const int TH = N / TW;
    p.TW = TW; p.tw_shift = TW == 8 ? 3 : (TW == 16 ? 4 : 5); p.N = N;
    p.tiles_x = cdiv(Wj, TW); p.tiles_y = cdiv(Hj, TH);
    p.n_patches = np;
    int rows = TH + max_off;
    const size_t wslot = 2 * (size_t)p.wtile_bytes;
    // a tall halo (large dilation) costs more than one box per tap, or does not fit: one patch per tap instead
    if (max_off > 0 && ((size_t)rows * TW * row_unit * 2 * 2 + 2 * wslot > 220 * 1024 || rows * np >= TH * ntaps)) {
        MS_REQUIRE(ntaps <= BF_MAX_PATCH, "conv_bf: too many per-tap patches");
        for (int i = 0; i < ntaps; ++i) {
            BfPatch& pt = p.patch[i];
            pt.dx = (short)taps[i].dx; pt.dy = (short)taps[i].dy; pt.tap0 = (short)i; pt.ntaps = 1;
            p.tap[i].row_off = 0; p.tap[i].widx = (short)taps[i].widx;
        }
        p.n_patches = ntaps;
        rows = TH;
    }
    MS_REQUIRE(rows * sx <= 256 && TW * sx <= 256, "conv_bf: patch too large for one TMA box");
    p.slot_bytes = (uint32_t)rows * TW * row_unit;
    const size_t pslot = 2 * (size_t)p.slot_bytes;
    const size_t budget = 220 * 1024;
    MS_REQUIRE(2 * pslot + 2 * wslot <= budget, "conv_bf: patch does not fit shared memory");
    int NP = 2, NW = 2;
    for (;;) {                                       // grow the two rings alternately while they fit (weights first: smaller)
        bool grew = false;
        if (NW < 8 && (size_t)NP * pslot + (size_t)(NW + 1) * wslot <= budget && NW <= 2 * NP) { ++NW; grew = true; }
        if (NP < 4 && (size_t)(NP + 1) * pslot + (size_t)NW * wslot <= budget) { ++NP; grew = true; }
        if (!grew) break;
    }
    p.NP = NP; p.NW = NW;
    p.y = g.y.p; p.ycs = g.y.cs; p.bias = g.bias; p.alpha = g.alpha;
    p.res = g.res; p.res_cs = g.res_cs; p.mask = g.mask; p.mask_cs = g.mask_cs; p.mask_alpha = g.mask_alpha;
    p.accumulate = g.accumulate;
    if (yp && yp->hi) {
        MS_REQUIRE(yp->cs >= M && (yp->cs & 7) == 0, "conv_bf: bad output planes");
        p.ohi = yp->hi; p.olo = yp->lo; p.ocs = yp->cs; p.ofmt = yp->fmt; p.oscale = yp->fmt == 1 ? yp->scale : 1.f;
    }
    p.wtiles = static_cast<const unsigned char*>(wtiles);
    // ---- split K over (K block, patch) units when the map is too small to fill the GPU (at most 8 ways: the closing
    //      CTA reads every partial sum).  The split is as wide as the idle SMs allow: the serial K loop of a grid of a few
    //      CTAs costs more than the partial-sum round trip.
    const int grid_tiles = p.NB * p.tiles_x * p.tiles_y;
    const int units = p.kblocks * p.n_patches;
    int ksplit = 1;
    if (part && tickets && (long)grid_tiles * mblocks <= NUM_SMS / 2 && units > 1) {
        ksplit = std::min(std::min(units, 8), std::max(1, NUM_SMS / (grid_tiles * mblocks)));
        while (ksplit > 1 && (size_t)ksplit * grid_tiles * mblocks * N * 128 > conv_bf_part_floats()) --ksplit;
        if ((size_t)grid_tiles * mblocks > conv_bf_ticket_words()) ksplit = 1;
    }
    p.ksplit = ksplit; p.part = part; p.tickets = tickets;

    const CUtensorMap *mXh, *mXl;
    {
        cuuint64_t dims[4] = {(cuuint64_t)g.x.c, (cuuint64_t)g.x.w, (cuuint64_t)g.x.h, (cuuint64_t)g.x.n};
        cuuint64_t strides[3] = {(cuuint64_t)xp.cs * 2, (cuuint64_t)g.x.w * xp.cs * 2, (cuuint64_t)g.x.h * g.x.w * xp.cs * 2};
        cuuint32_t box[4] = {(cuuint32_t)p.kch, (cuuint32_t)(TW * sx), (cuuint32_t)(rows * sx), 1};
        cuuint32_t es[4] = {1, (cuuint32_t)sx, (cuuint32_t)sx, 1};
        if (bf_get_map(&mXh, xp.hi, 4, dims, strides, box, es, p.kch == 64 ? 128 : 64)) return -1;
        if (bf_get_map(&mXl, xp.lo, 4, dims, strides, box, es, p.kch == 64 ? 128 : 64)) return -1;
    }
    // the epilogue stages the accumulators in the ring buffers
    const size_t smem = std::max((size_t)NP * pslot + (size_t)NW * wslot, (size_t)N * BF_STAGE_LD * 4) + 1024;
    const dim3 grid(grid_tiles, mblocks, ksplit);
    const bool bf = xp.fmt == 0;
    if (N == 64) launch_k(bf ? conv_bf_kernel<64, 1> : conv_bf_kernel<64, 0>, grid, dim3(BF_THREADS), smem, st, *mXh, *mXl, p);
    else if (N == 96) launch_k(bf ? conv_bf_kernel<96, 1> : conv_bf_kernel<96, 0>, grid, dim3(BF_THREADS), smem, st, *mXh, *mXl, p);
    else launch_k(bf ? conv_bf_kernel<128, 1> : conv_bf_kernel<128, 0>, grid, dim3(BF_THREADS), smem, st, *mXh, *mXl, p);
    return check_launch("conv_bf");
}

// xp: 16-bit planes of g.x;  wtiles: prepared weight tiles in the SAME format as xp;  yp: optional planes of g.y (written
// by the epilogue in yp->fmt)
int conv_bf(const ConvGemm& g, const ActPlanes& xp, const void* wtiles, const ActPlanes* yp,
            float* part, unsigned int* tickets, cudaStream_t st) {
    MS_REQUIRE(conv_bf_supported(g), "conv_bf: unsupported geometry");
    MS_REQUIRE(xp.hi && xp.lo && (xp.cs & 7) == 0 && xp.cs >= g.x.c, "conv_bf: input planes missing");
    if (conv_bf_init()) return -1;
    const int taps_total = g.kh * g.kw;
    BfTapSpec taps[BF_MAX_TAPS];
    if (g.div == 1) {
        // gathered input pixel = out * mul + off + tap * step
        int n = 0;
        for (int s = 0; s < g.kw; ++s)
            for (int r = 0; r < g.kh; ++r) taps[n++] = BfTapSpec{g.off_y + r * g.step, g.off_x + s * g.step, r * g.kw + s};
        return conv_bf_launch(g, xp, wtiles, yp, part, tickets, g.y.h, g.y.w, 1, 0, 0, g.mul, taps, n, taps_total, st);
    }
    // fractionally strided gather (stride-2 dgrad, conv_transpose): t = out + off + tap*step must be even, input = t / 2.
    // Output pixels of one parity class (py, px) see a fixed subset of the taps at unit input stride: four dense launches.
    for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
            const int Hj = (g.y.h - py + 1) / 2, Wj = (g.y.w - px + 1) / 2;
            if (Hj <= 0 || Wj <= 0) continue;
            int n = 0;
            for (int s = 0; s < g.kw; ++s) {
                const int tx = px + g.off_x + s * g.step;
                if (tx & 1) continue;
                for (int r = 0; r < g.kh; ++r) {
                    const int ty = py + g.off_y + r * g.step;
                    if (ty & 1) continue;
                    taps[n++] = BfTapSpec{ty / 2, tx / 2, r * g.kw + s};    // exact: ty, tx even (C++ division truncates toward 0)
                }
            }
            if (n == 0) { set_error("conv_bf: parity class without taps"); return -2; }
            if (conv_bf_launch(g, xp, wtiles, yp, part, tickets, Hj, Wj, 2, py, px, 1, taps, n, taps_total, st)) return -1;
        }
    return 0;
}

// one-shot convenience (operator-level C ABI / tests): splits the input, prepares the weights, runs the conv.
//   fmt: operand format (1 = fp16 forward planes, 0 = bf16 gradient planes)
//   scratch layout (bytes): [x hi | x lo | weight tiles | job | tickets | split-K partials]
size_t conv_bf_oneshot_scratch_bytes(const ConvGemm& g) {
    const size_t xe = g.x.pixels() * ((g.x.c + 7) / 8 * 8);
    const size_t we = conv_bf_weight_halfs(g.kh * g.kw, g.y.c, g.x.c);
    return 2 * (xe * 2 + 256) + (we * 2 + 256) + 1024 + conv_bf_ticket_words() * 4 + conv_bf_part_floats() * 4 + 4096;
}

int conv_bf_oneshot(const ConvGemm& g, int wmat_is_mk, int fmt, float act_scale, void* scratch, size_t scratch_bytes, cudaStream_t st) {
    MS_REQUIRE(conv_bf_supported(g), "conv_bf: unsupported geometry");
    MS_REQUIRE(scratch_bytes >= conv_bf_oneshot_scratch_bytes(g), "conv_bf: scratch too small");
    MS_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, "conv_bf: scratch must be 256B aligned");
    unsigned char* b = reinterpret_cast<unsigned char*>(scratch);
    auto take = [&](size_t bytes) { unsigned char* r = b; b += (bytes + 255) / 256 * 256; return r; };
    const int pcs = (g.x.c + 7) / 8 * 8;
    const size_t xe = g.x.pixels() * pcs;
    const size_t we = conv_bf_weight_halfs(g.kh * g.kw, g.y.c, g.x.c);
    ActPlanes xp; xp.hi = take(xe * 2); xp.lo = take(xe * 2); xp.cs = pcs; xp.fmt = fmt; xp.scale = fmt == 1 ? act_scale : 1.f;
    void* wt = take(we * 2);
    BfPrepJob* jd = reinterpret_cast<BfPrepJob*>(take(1024));
    unsigned int* tickets = reinterpret_cast<unsigned int*>(take(conv_bf_ticket_words() * 4));
    float* part = reinterpret_cast<float*>(take(conv_bf_part_floats() * 4));
    int Mpad, Kpad; conv_bf_weight_dims(g.y.c, g.x.c, Mpad, Kpad);
    BfPrepJob job{g.wmat, wt, g.kh * g.kw, g.y.c, g.x.c, Mpad, Kpad, wmat_is_mk ? 0 : 1, fmt};
    MS_CHECK_CUDA(cudaMemcpyAsync(jd, &job, sizeof job, cudaMemcpyHostToDevice, st));
    MS_CHECK_CUDA(cudaMemsetAsync(tickets, 0, conv_bf_ticket_words() * 4, st));
    if (bf_prep_weights(jd, 1, we, st)) return -1;
    if (split_planes(g.x, xp, st)) return -1;
    return conv_bf(g, xp, wt, nullptr, part, tickets, st);
}

}  // namespace ms
