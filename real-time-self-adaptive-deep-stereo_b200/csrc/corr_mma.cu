// Wide-window horizontal correlation (DispNet: 81 displacements, 128 channels) as a banded product on the warp-level
// tensor-core path.
//
// Replaces sharedLayers.correlation for the DispNet-C call site (reference Nets/DispNet.py:92-101 -> Nets/sharedLayers.py:23-51,
// max_disp = 40, stride 1, no warp):
//     corr[b,y,x,i] = (1/C) * sum_c L[b,y,x,c] * R[b,y,x+i-D,c]          0 <= i <= 2D, zero outside the row
// For one image row this is the band |x' - x| <= D of the w x w matrix L R^T.  The narrow-window kernels (corr.cu,
// corr_tma.cu: 5 displacements) keep one pixel per 8 lanes and are bandwidth-shaped; at 81 displacements the same loop is
// arithmetic-bound on the CUDA cores (0.64 GFLOP of scalar FMAs with one shared-memory operand each at 1280x384,
// 4.4 % of the HBM roofline).  Here a warp owns a 16-pixel block of x and the 16 + 2D window of x' it can reach:
// 12 m16n8k16 tiles per K step for D = 40, 84 % of the multiplied entries inside the band.
//
// Why mma.sync: the result has to be read along DIAGONALS (i = x' - x + D).  In the mma.sync accumulator fragment a
// thread owns fixed (row, column) pairs, so i = col - row is a per-register constant and the band is extracted with no
// data movement.
// The op is 2 GFLOP of issued MMAs against 41 MB of HBM traffic -- the HBM roofline, not the tensor pipe, is the bound.
//
// Arithmetic: fp32 features are split while they are staged into shared memory, x * s = hi + lo in fp16 (22 mantissa
// bits, s = the engine's power-of-two activation scale), three MMAs per product (hi*hi + hi*lo + lo*hi) accumulated in
// fp32 -- the same scheme as the forward convolutions (conv_bf.cu).
#include "common.cuh"
#include <algorithm>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace ms {

constexpr int CM_TX = 64;          // pixels of x per CTA (4 m16 blocks)
constexpr int CM_KC = 64;          // channels per staged chunk
constexpr int CM_PITCH = CM_KC + 8;   // halfs per smem row: 144 B, ldmatrix rows land in distinct banks
constexpr int CM_NT = 256;
constexpr int CM_MAXD = 40;
constexpr int CM_TILES_W = 6;      // n8 tiles per warp (two warps share an m block: 12 tiles = 96 columns)

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_f16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split_f16(float v, float s, unsigned short& h, unsigned short& l) {
    const float t = v * s;
    unsigned short hh, ll;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(hh) : "f"(t));
    const float r = t - __half2float(__ushort_as_half(hh));
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(ll) : "f"(r));
    h = hh; l = ll;
}

// grid (ceil(w / 64), B * h); smem: [L hi | L lo | R hi | R lo] rows of CM_PITCH halfs, reused as the fp32 output stage
__global__ void __launch_bounds__(CM_NT, 2) corr_mma_kernel(CorrFwd p, int nd, int ntl, int rrows, float scale, float inv) {
    pdl_prologue();
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int C = p.C, w = p.w, D = p.max_disp;
    const int row = blockIdx.y, x0 = blockIdx.x * CM_TX;
    unsigned short* Lh = reinterpret_cast<unsigned short*>(smem_raw);
    unsigned short* Ll = Lh + CM_TX * CM_PITCH;
    unsigned short* Rh = Ll + CM_TX * CM_PITCH;
    unsigned short* Rl = Rh + (size_t)rrows * CM_PITCH;
    const float* lrow = p.left + (size_t)row * w * p.lcs;
    const float* rrow = p.right + (size_t)row * w * p.rcs;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mb = warp >> 1, nh = warp & 1;          // m block (16 pixels of x), half of its window tiles
    const int g = lane >> 2, t = lane & 3;
    float acc[CM_TILES_W][4];
#pragma unroll
    for (int j = 0; j < CM_TILES_W; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }

    // ldmatrix lane addresses (element offsets inside a plane)
    //   A (16 x 16 of L): lanes 0-7 rows 0-7 k 0-7 | 8-15 rows 8-15 k 0-7 | 16-23 rows 0-7 k 8-15 | 24-31 rows 8-15 k 8-15
    const int a_row = mb * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, a_k = (lane >> 4) * 8;
    //   B (two n8 tiles of R^T): lanes 0-7 n 0-7 k 0-7 | 8-15 n 0-7 k 8-15 | 16-23 n 8-15 k 0-7 | 24-31 n 8-15 k 8-15
    const int b_row = mb * 16 + nh * (CM_TILES_W * 8) + (lane & 7) + (lane >> 4) * 8, b_k = ((lane >> 3) & 1) * 8;
    const uint32_t sLh = (uint32_t)__cvta_generic_to_shared(Lh), sLl = (uint32_t)__cvta_generic_to_shared(Ll);
    const uint32_t sRh = (uint32_t)__cvta_generic_to_shared(Rh), sRl = (uint32_t)__cvta_generic_to_shared(Rl);

    for (int c0 = 0; c0 < C; c0 += CM_KC) {
        const int kc = min(CM_KC, C - c0);           // multiple of 16 (checked by the host)
        const int nq = CM_KC / 4;
        if (c0) __syncthreads();                     // the previous chunk's fragments are consumed
        // ---- stage + split: L rows [x0, x0 + 64), R rows [x0 - D, x0 - D + rrows); zeros outside the image row / chunk
        for (int e = threadIdx.x; e < (CM_TX + rrows) * nq; e += CM_NT) {
            const int px = e / nq, q = e - px * nq;
            const bool isL = px < CM_TX;
            const int x = isL ? x0 + px : x0 - D + (px - CM_TX);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (x >= 0 && x < w && q * 4 < kc)
                v = __ldg(reinterpret_cast<const float4*>((isL ? lrow + (size_t)x * p.lcs : rrow + (size_t)x * p.rcs) + c0 + q * 4));
            unsigned short h[4], l[4];
            split_f16(v.x, scale, h[0], l[0]); split_f16(v.y, scale, h[1], l[1]);
            split_f16(v.z, scale, h[2], l[2]); split_f16(v.w, scale, h[3], l[3]);
            uint2 hv, lv;
            hv.x = (uint32_t)h[0] | ((uint32_t)h[1] << 16); hv.y = (uint32_t)h[2] | ((uint32_t)h[3] << 16);
            lv.x = (uint32_t)l[0] | ((uint32_t)l[1] << 16); lv.y = (uint32_t)l[2] | ((uint32_t)l[3] << 16);
            const int r = isL ? px : px - CM_TX;
            unsigned short* dh = (isL ? Lh : Rh) + (size_t)r * CM_PITCH + q * 4;
            unsigned short* dl = (isL ? Ll : Rl) + (size_t)r * CM_PITCH + q * 4;
            *reinterpret_cast<uint2*>(dh) = hv;
            *reinterpret_cast<uint2*>(dl) = lv;
        }
        __syncthreads();
        // ---- banded product of this chunk
        for (int ks = 0; ks < kc; ks += 16) {
            uint32_t ah[4], al[4];
            const uint32_t aoff = (uint32_t)(a_row * CM_PITCH + ks + a_k) * 2u;
            ldsm_x4(sLh + aoff, ah[0], ah[1], ah[2], ah[3]);
            ldsm_x4(sLl + aoff, al[0], al[1], al[2], al[3]);
#pragma unroll
            for (int jp = 0; jp < CM_TILES_W / 2; ++jp) {
                if (nh * CM_TILES_W + 2 * jp >= ntl) continue;      // (warp-uniform: narrower windows use fewer tiles)
                uint32_t bh[4], bl[4];
                const uint32_t boff = (uint32_t)((b_row + jp * 16) * CM_PITCH + ks + b_k) * 2u;
                ldsm_x4(sRh + boff, bh[0], bh[1], bh[2], bh[3]);
                ldsm_x4(sRl + boff, bl[0], bl[1], bl[2], bl[3]);
                mma_f16(acc[2 * jp], al, bh[0], bh[1]);
                mma_f16(acc[2 * jp], ah, bl[0], bl[1]);
                mma_f16(acc[2 * jp], ah, bh[0], bh[1]);
                mma_f16(acc[2 * jp + 1], al, bh[2], bh[3]);
                mma_f16(acc[2 * jp + 1], ah, bl[2], bl[3]);
                mma_f16(acc[2 * jp + 1], ah, bh[2], bh[3]);
            }
        }
    }
    __syncthreads();
    // ---- band extraction: accumulator (r, col) of m block mb is L[x0 + 16 mb + r] . R[x0 + 16 mb - D + col]: i = col - r
    float* S = reinterpret_cast<float*>(smem_raw);       // [64][nd]
#pragma unroll
    for (int j = 0; j < CM_TILES_W; ++j) {
        const int colb = (nh * CM_TILES_W + j) * 8 + 2 * t;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int r = g + (e >> 1) * 8, col = colb + (e & 1);
            const int i = col - r;
            if (i >= 0 && i < nd) S[(mb * 16 + r) * nd + i] = acc[j][e] * inv;
        }
    }
    __syncthreads();
    const int coff = p.copy_left ? C : 0;
    float* orow = p.out + (size_t)row * w * p.ocs + coff;
    const int npx = min(CM_TX, w - x0);
    for (int e = threadIdx.x; e < npx * nd; e += CM_NT) {
        const int px = e / nd, i = e - px * nd;
        orow[(size_t)(x0 + px) * p.ocs + i] = S[e];
    }
}

bool corr_mma_supported(const CorrFwd& p) {
    const int nd = 2 * p.max_disp / std::max(p.stride, 1) + 1;
    return p.u == nullptr && p.stride == 1 && p.plane_scale > 0.f && p.max_disp <= CM_MAXD && nd >= 17 && (p.C % 16) == 0 &&
           !p.copy_left && (p.lcs % 4) == 0 && (p.rcs % 4) == 0 && ((reinterpret_cast<uintptr_t>(p.left) | reinterpret_cast<uintptr_t>(p.right)) & 15) == 0;
}

int corr_mma(const CorrFwd& p, cudaStream_t st) {
    MS_REQUIRE(corr_mma_supported(p), "corr_mma: unsupported geometry");
    const int D = p.max_disp, nd = 2 * D + 1;
    const int ntl = (16 + 2 * D + 7) / 8;                  // window tiles per m block (12 for D = 40)
    const int rrows = 48 + 2 * CM_TILES_W * 8;             // rows the ldmatrix addresses can touch (tiles beyond ntl are skipped, not read)
    const size_t smem = (size_t)(CM_TX + rrows) * CM_PITCH * 2 * 2;
    MS_REQUIRE(smem >= (size_t)CM_TX * nd * 4, "corr_mma: output stage does not fit");
    static bool init = false;
    if (!init) {
        MS_CHECK_CUDA(cudaFuncSetAttribute(corr_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        init = true;
    }
    const float inv = 1.f / ((float)p.C * p.plane_scale * p.plane_scale);
    launch_k(corr_mma_kernel, dim3(cdiv(p.w, CM_TX), p.B * p.h), dim3(CM_NT), smem, st, p, nd, ntl, rrows, p.plane_scale, inv);
    return check_launch("corr_mma");
}


// ------------------------------------------------------------------------------------------------
// backward: the two gradients are banded products with the gradient band G[x][x'] = g[x][x' - x + D] in the A role
//     dL[x , :] = (1/C) sum_{x'} G[x][x'] R[x', :]          (role 0)
//     dR[x', :] = (1/C) sum_{x }  G[x][x'] L[x , :]          (role 1)
// For a 16-pixel block starting at X both read a 96-row window (rows X - D ... X - D + 95) of the other feature map:
//     A[r][col] = g[X + r][col - r]                 role 0,      A[r][col] = g[X - D + col][2D - (col - r)]      role 1
// (zero where the displacement index leaves [0, nd)), M = 16, K = 96 window rows, N = C channels.  Operands are bf16 hi/lo
// (gradients have no usable fixed scale; same 3-MMA scheme as the convolution gradients, ~2^-17 relative per product).
// B fragments come from the [row][channel] window through ldmatrix.trans.
// ------------------------------------------------------------------------------------------------
constexpr int CB_K = 96;                // window rows = K of the product
constexpr int CB_APITCH = CB_K + 8;     // halfs per row of the A image (208 B: ldmatrix rows in distinct banks)

__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split_bf16(float v, unsigned short& h, unsigned short& l) {
    const __nv_bfloat16 hb = __float2bfloat16_rn(v);
    h = __bfloat16_as_ushort(hb);
    l = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(hb)));
}

// grid (ceil(w / 64), B * h, 2 roles); smem: [A hi | A lo] 64 x CB_APITCH, [W hi | W lo] 144 x (C + 8)
__global__ void __launch_bounds__(CM_NT, 2) corr_mma_bwd_kernel(CorrBwd p, int nd, int gc, float inv) {
    pdl_prologue();
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int C = p.C, w = p.w, D = p.max_disp;
    const int role = blockIdx.z;
    const int row = blockIdx.y, x0 = blockIdx.x * CM_TX;
    const int wpitch = C + 8;
    constexpr int WROWS = 48 + CB_K;
    unsigned short* Ah = reinterpret_cast<unsigned short*>(smem_raw);
    unsigned short* Al = Ah + CM_TX * CB_APITCH;
    unsigned short* Wh = Al + CM_TX * CB_APITCH;
    unsigned short* Wl = Wh + (size_t)WROWS * wpitch;
    const float* grow = p.dcost + (size_t)row * w * p.dcs + gc;
    const float* frow = role == 0 ? p.right + (size_t)row * w * p.rcs : p.left + (size_t)row * w * p.lcs;
    const int fcs = role == 0 ? p.rcs : p.lcs;

    // ---- the gradient band as the A operand (gathered straight from global: 41 KB per CTA, L2 resident)
    for (int e = threadIdx.x; e < CM_TX * CB_K; e += CM_NT) {
        const int rr = e / CB_K, col = e - rr * CB_K;          // rr = 16 * mb + r
        const int r = rr & 15, X = x0 + (rr & ~15);
        const int xa = role == 0 ? X + r : X - D + col;
        const int ia = role == 0 ? col - r : 2 * D - (col - r);
        float v = 0.f;
        if (ia >= 0 && ia < nd && xa >= 0 && xa < w) v = __ldg(grow + (size_t)xa * p.dcs + ia);
        unsigned short h, l;
        split_bf16(v, h, l);
        Ah[rr * CB_APITCH + col] = h;
        Al[rr * CB_APITCH + col] = l;
    }
    // ---- the feature window rows x0 - D ... x0 - D + 143 as the B operand
    const int nq = C / 4;
    for (int e = threadIdx.x; e < WROWS * nq; e += CM_NT) {
        const int rr = e / nq, q = e - rr * nq;
        const int x = x0 - D + rr;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x >= 0 && x < w) v = __ldg(reinterpret_cast<const float4*>(frow + (size_t)x * fcs + q * 4));
        unsigned short h[4], l[4];
        split_bf16(v.x, h[0], l[0]); split_bf16(v.y, h[1], l[1]); split_bf16(v.z, h[2], l[2]); split_bf16(v.w, h[3], l[3]);
        uint2 hv, lv;
        hv.x = (uint32_t)h[0] | ((uint32_t)h[1] << 16); hv.y = (uint32_t)h[2] | ((uint32_t)h[3] << 16);
        lv.x = (uint32_t)l[0] | ((uint32_t)l[1] << 16); lv.y = (uint32_t)l[2] | ((uint32_t)l[3] << 16);
        *reinterpret_cast<uint2*>(Wh + (size_t)rr * wpitch + q * 4) = hv;
        *reinterpret_cast<uint2*>(Wl + (size_t)rr * wpitch + q * 4) = lv;
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mb = warp >> 1, nh = warp & 1;          // m block; half of the channels
    const int g = lane >> 2, t = lane & 3;
    const int ntw = C / 16;                           // n8 tiles of this warp (C / 2 channels), even
    float acc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
    const int a_row = mb * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, a_k = (lane >> 4) * 8;
    // B through ldmatrix.trans on [k row][channel]: lanes 0-7 k 0-7 n 0-7 | 8-15 k 8-15 n 0-7 | 16-23 k 0-7 n 8-15 | 24-31 k 8-15 n 8-15
    const int b_krow = mb * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, b_n = nh * (C / 2) + (lane >> 4) * 8;
    const uint32_t sAh = (uint32_t)__cvta_generic_to_shared(Ah), sAl = (uint32_t)__cvta_generic_to_shared(Al);
    const uint32_t sWh = (uint32_t)__cvta_generic_to_shared(Wh), sWl = (uint32_t)__cvta_generic_to_shared(Wl);
    for (int ks = 0; ks < CB_K; ks += 16) {
        uint32_t ah[4], al[4];
        const uint32_t aoff = (uint32_t)(a_row * CB_APITCH + ks + a_k) * 2u;
        ldsm_x4(sAh + aoff, ah[0], ah[1], ah[2], ah[3]);
        ldsm_x4(sAl + aoff, al[0], al[1], al[2], al[3]);
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
            if (2 * jp >= ntw) continue;
            uint32_t bh[4], bl[4];
            const uint32_t boff = (uint32_t)((b_krow + ks) * wpitch + b_n + jp * 16) * 2u;
            ldsm_x4_t(sWh + boff, bh[0], bh[1], bh[2], bh[3]);
            ldsm_x4_t(sWl + boff, bl[0], bl[1], bl[2], bl[3]);
            mma_bf16(acc[2 * jp], al, bh[0], bh[1]);
            mma_bf16(acc[2 * jp], ah, bl[0], bl[1]);
            mma_bf16(acc[2 * jp], ah, bh[0], bh[1]);
            mma_bf16(acc[2 * jp + 1], al, bh[2], bh[3]);
            mma_bf16(acc[2 * jp + 1], ah, bl[2], bl[3]);
            mma_bf16(acc[2 * jp + 1], ah, bh[2], bh[3]);
        }
    }
    // ---- epilogue: accumulator (r, n) -> d(feature)[x0 + 16 mb + r][n]; 8-byte stores, one full sector per row and tile
    float* orow = role == 0 ? p.dleft + (size_t)row * w * p.dlcs : p.dright + (size_t)row * w * p.drcs;
    const int ocs = role == 0 ? p.dlcs : p.drcs;
    const bool accum = role == 0 ? p.acc_left != 0 : p.acc_right != 0;
    const bool add_slice = role == 0 && p.add_left_slice;
    const float* srow = p.dcost + (size_t)row * w * p.dcs;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (j >= ntw) continue;
        const int n = nh * (C / 2) + j * 8 + 2 * t;
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int x = x0 + mb * 16 + g + hrow * 8;
            if (x >= w) continue;
            float2 v = make_float2(acc[j][2 * hrow] * inv, acc[j][2 * hrow + 1] * inv);
            float2* dst = reinterpret_cast<float2*>(orow + (size_t)x * ocs + n);
            if (add_slice) { const float2 sl = *reinterpret_cast<const float2*>(srow + (size_t)x * p.dcs + n); v.x += sl.x; v.y += sl.y; }
            if (accum) { const float2 o = *dst; v.x += o.x; v.y += o.y; }
            *dst = v;
        }
    }
}

bool corr_mma_bwd_supported(const CorrBwd& p) {
    const int nd = 2 * p.max_disp / std::max(p.stride, 1) + 1;
    return p.u == nullptr && p.du == nullptr && p.stride == 1 && p.max_disp <= CM_MAXD && nd >= 17 && (p.C % 32) == 0 && p.C <= 128 &&
           (p.lcs % 4) == 0 && (p.rcs % 4) == 0 && (p.dlcs % 2) == 0 && (p.drcs % 2) == 0 && (!p.add_left_slice || (p.dcs % 2) == 0) &&
           ((reinterpret_cast<uintptr_t>(p.left) | reinterpret_cast<uintptr_t>(p.right)) & 15) == 0 &&
           ((reinterpret_cast<uintptr_t>(p.dleft) | reinterpret_cast<uintptr_t>(p.dright) | reinterpret_cast<uintptr_t>(p.dcost)) & 7) == 0;
}

int corr_mma_bwd(const CorrBwd& p, cudaStream_t st) {
    MS_REQUIRE(corr_mma_bwd_supported(p), "corr_mma_bwd: unsupported geometry");
    const int nd = 2 * p.max_disp + 1;
    const int gc = p.gcoff < 0 ? p.C : p.gcoff;
    const size_t smem = (size_t)CM_TX * CB_APITCH * 2 * 2 + (size_t)(48 + CB_K) * (p.C + 8) * 2 * 2;
    static size_t attr = 0;
    if (smem > attr) {
        MS_CHECK_CUDA(cudaFuncSetAttribute(corr_mma_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    launch_k(corr_mma_bwd_kernel, dim3(cdiv(p.w, CM_TX), p.B * p.h, 2), dim3(CM_NT), smem, st, p, nd, gc, 1.f / (float)p.C);
    return check_launch("corr_mma_bwd");
}

}  // namespace ms
