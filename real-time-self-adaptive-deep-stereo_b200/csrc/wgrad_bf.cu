// wgrad_bf: wgmma weight (+ bias) gradient of a convolution on split-bf16 operands, stride 1 or 2, any dilation.
//
// Replaces the filter- and bias-gradient sub-graphs tf.gradients derives for tf.nn.conv2d / tf.nn.atrous_conv2d /
// tf.nn.bias_add (reference Nets/sharedLayers.py:58-59,72-73) inside the train ops of
// Stereo_Online_Adaptation.py:118,128.
//
//   dW[r][s][ci][co] = sum over output pixels p of  X[p * stride + offset(r, s)][ci] * dY[p][co]
//   db[co]           = sum over output pixels p of  dY[p][co]
//
// Both operands already exist as 16-bit hi / lo planes in NHWC (the forward activation planes conv_bf reads, and the
// gradient planes the dgrad epilogue writes), i.e. with the GEMM's reduction index (pixels) as the SLOW index.  The wgmma
// descriptors take that layout directly as "MN-major" operands: a TMA box {64 channels, 8 pixels, rows} with
// SWIZZLE_128B is exactly the canonical MN-major SW128 tile ((8,n),(8,k)):((1,LBO),(8,SBO)) [uint128 units] with
// SBO = 1024 B (8 pixels) and LBO = the distance between 64-channel blocks -- no transposes, no in-kernel splitting.
//
// GEMM per CTA: one filter COLUMN s (all kh <= 3 taps of it: one register accumulator per tap), one 128-row block of ci
// (two warpgroups of m64 wgmma), one block of WB_BN = 64 output channels, one slice of the pixel tiles (split-K):
//   M = ci, N = co, K = pixels in tiles of 8 x TH.
//   For stride 1 and small dilation the kh taps read ONE halo patch of X (TH + (kh-1)*dil rows; a tap is a row offset =
//   a whole number of 1024-byte swizzle atoms = a different descriptor start address); otherwise one box per tap
//   (stride 2 through TMA element strides).
//   Three 16-bit MMAs per K step: X_lo*dY_hi + X_hi*dY_lo + X_hi*dY_hi (~2^-16 relative product error).
//   Bias gradient: CTAs of column 0 / block 0 run two more MMAs per K step with an all-ones A tile -> db in one more
//   accumulator (no separate reduction kernel over dY).
// Partial sums [split][tap][ci][co] (+ [split][co]) go to the workspace; a fixed-order reduce finishes (deterministic).
//
// Warpgroup roles (384 threads): warpgroup 0 = TMA producer (one warp issues), warpgroups 1-2 = wgmma on ci [0, 64) /
// [64, 128) of the block, then they store their partial sums straight from the accumulator registers.
#include <cuda.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace ms {

constexpr int WB_THREADS = 384;
constexpr int WB_MAX_KH = 7;
constexpr int WB_ACC_TAPS = 3;                 // filter rows per launch: 3 tap accumulators + the bias accumulator
constexpr int WB_BN = 64;                      // output channels per CTA
constexpr uint32_t WB_ONES_BYTES = 4096;       // 2 channel blocks x 2 k-groups x 1024 B of 1.0
constexpr uint32_t WB_ATOM = 1024;             // one tile row: 8 pixels x 64 channels x 2 B

struct WgradBfParams {
    int kh, kw;
    int tiles_x, tiles_y, ntiles, splits;
    int TH;                        // pixel tile = 8 wide x TH high (TH even)
    int sx;                        // forward stride: input pixel = out * sx + offset
    int nbox, box_rows, x_rows;    // X boxes per 64-channel block and plane; tile rows per box; rows of the X region
    short box_dy[WB_MAX_KH];       // input-row origin of box b relative to y0 * sx
    short tap_row[WB_MAX_KH];      // first X-region row of tap r
    int pad_l, dil;
    int ci, co, mblocks, nblocks, xblk;
    int nstages;
    uint32_t stage_bytes, x_plane_bytes, d_plane_bytes;
    int with_bias;
    float* part;                   // [split][tap][ci][co]
    float* bpart;                  // [split][co]
    int tap0, taps_total;          // this launch covers filter rows [tap0 / kw, tap0 / kw + kh) of a taps_total-tap filter
};

// BF: 1 = bf16 planes, 0 = fp16 planes (both operands share the format: a wgmma takes one A / B element type)
template <int BF>
__global__ void __launch_bounds__(WB_THREADS, 1)
wgrad_bf_kernel(const __grid_constant__ CUtensorMap mapXh, const __grid_constant__ CUtensorMap mapXl,
                const __grid_constant__ CUtensorMap mapDh, const __grid_constant__ CUtensorMap mapDl,
                const __grid_constant__ WgradBfParams p) {
    pdl_prologue();
    extern __shared__ unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t full_bar[4], empty_bar[4];

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const uint32_t base = (s_addr(smem_dyn) + 1023u) & ~1023u;
    unsigned char* gbase = smem_dyn + (base - s_addr(smem_dyn));
    const uint32_t stage0 = WB_ONES_BYTES;

    int bx = blockIdx.x;
    const int nb = bx % p.nblocks; bx /= p.nblocks;
    const int mb = bx % p.mblocks;
    const int s = bx / p.mblocks;                       // filter column
    const int split = blockIdx.y;
    const int t0 = (int)(((long)split * p.ntiles) / p.splits), t1 = (int)(((long)(split + 1) * p.ntiles) / p.splits);
    const bool do_bias = p.with_bias && s == 0 && mb == 0;

    if (threadIdx.x == 0) {
        // full: the producer's expect_tx arrival + the bytes; empty: one arrival per MMA warp (8)
        for (int i = 0; i < p.nstages; ++i) { mb_init(&full_bar[i], 1); mb_init(&empty_bar[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp >= 4) {                                    // the all-ones A tile of the bias-gradient MMAs
        uint32_t* ones = reinterpret_cast<uint32_t*>(gbase);
        const uint32_t one2 = BF ? 0x3F803F80u : 0x3C003C00u;      // 1.0 in the format of the dY planes
        for (int i = threadIdx.x - 128; i < (int)(WB_ONES_BYTES / 4); i += WB_THREADS - 128) ones[i] = one2;
        fence_async_smem();
    }
    __syncthreads();

    if (warp < 4) {
        // ================= TMA producer: warp-uniform loop, elected lane issues =================
        if (warp == 0) {
            const bool leader = elect_one();
            int st = 0; uint32_t ph = 0;
            const int tiles_img = p.tiles_x * p.tiles_y;
            const int offx = s * p.dil - p.pad_l;
            for (int t = t0; t < t1; ++t) {
                const int img = t / tiles_img;
                const int rem = t - img * tiles_img;
                const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
                mb_wait(&empty_bar[st], ph ^ 1u);
                if (leader) mb_expect_tx(&full_bar[st], p.stage_bytes);
                unsigned char* dst = gbase + stage0 + (size_t)st * p.stage_bytes;
                for (int pl = 0; pl < 2 && leader; ++pl) {
                    const CUtensorMap* mx = pl ? &mapXl : &mapXh;
                    unsigned char* xd = dst + (size_t)pl * p.x_plane_bytes;
                    for (int b = 0; b < p.xblk; ++b)
                        for (int q = 0; q < p.nbox; ++q)
                            tma_load_4d(xd + (size_t)(b * p.x_rows + q * p.box_rows) * WB_ATOM, mx, &full_bar[st],
                                        mb * 128 + b * 64, tx * 8 * p.sx + offx, ty * p.TH * p.sx + p.box_dy[q], img);
                    const CUtensorMap* md = pl ? &mapDl : &mapDh;
                    unsigned char* dd = dst + 2 * (size_t)p.x_plane_bytes + (size_t)pl * p.d_plane_bytes;
                    tma_load_4d(dd, md, &full_bar[st], nb * WB_BN, tx * 8, ty * p.TH, img);
                }
                if (++st == p.nstages) { st = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ================= MMA warpgroups: ci rows [64 * mg, 64 * mg + 64) of the block =================
    const int mg = (warp >> 2) - 1;
    const bool rows_live = mg < p.xblk;                 // (ci <= 64: the second warpgroup has no rows, only the bias MMAs run)
    const bool bias_here = do_bias && mg == 0;
    float acc[WB_ACC_TAPS][WB_BN / 2], accb[WB_BN / 2];
#pragma unroll
    for (int i = 0; i < WB_BN / 2; ++i) {
        accb[i] = 0.f;
#pragma unroll
        for (int r = 0; r < WB_ACC_TAPS; ++r) acc[r][i] = 0.f;
    }
    {
        const uint32_t x_rows_bytes = (uint32_t)p.x_rows * WB_ATOM;
        const uint64_t ones = wg_desc(base, 2048u, 1024u, true);
        int st = 0; uint32_t ph = 0;
        int pend = -1;                                  // ring stage read by the MMAs still in flight
        const int ksteps = p.TH >> 1;
        for (int t = t0; t < t1; ++t) {
            mb_wait(&full_bar[st], ph);
            const uint32_t sb = base + stage0 + (uint32_t)st * p.stage_bytes;
            const uint32_t xh = sb + (uint32_t)mg * x_rows_bytes, xl = xh + p.x_plane_bytes;
            const uint32_t dh = sb + 2u * p.x_plane_bytes, dl = dh + p.d_plane_bytes;
#pragma unroll
            for (int r = 0; r < WB_ACC_TAPS; ++r) wg_fence_acc(acc[r]);
            wg_fence_acc(accb);
            wg_fence();
            for (int j = 0; j < ksteps; ++j) {          // K = 16 pixels = two 8-pixel atoms
                const uint64_t bh = wg_desc(dh + (uint32_t)(2 * j) * WB_ATOM, 0u, 1024u, true);
                const uint64_t bl = wg_desc(dl + (uint32_t)(2 * j) * WB_ATOM, 0u, 1024u, true);
                if (rows_live) {
#pragma unroll
                    for (int r = 0; r < WB_ACC_TAPS; ++r) {
                        if (r >= p.kh) break;
                        const uint32_t ro = (uint32_t)(p.tap_row[r] + 2 * j) * WB_ATOM;
                        const uint64_t ah = wg_desc(xh + ro, 0u, 1024u, true);
                        const uint64_t al = wg_desc(xl + ro, 0u, 1024u, true);
                        Wgmma<WB_BN, BF, 1, 1>::mma(acc[r], al, bh);
                        Wgmma<WB_BN, BF, 1, 1>::mma(acc[r], ah, bl);
                        Wgmma<WB_BN, BF, 1, 1>::mma(acc[r], ah, bh);
                    }
                }
                if (bias_here) {
                    Wgmma<WB_BN, BF, 1, 1>::mma(accb, ones, bl);
                    Wgmma<WB_BN, BF, 1, 1>::mma(accb, ones, bh);
                }
            }
            wg_commit();
            wg_wait<1>();                               // the previous stage's MMAs are done with their operands
#pragma unroll
            for (int r = 0; r < WB_ACC_TAPS; ++r) wg_fence_acc(acc[r]);
            wg_fence_acc(accb);
            if (pend >= 0 && lane == 0) mb_arrive(&empty_bar[pend]);
            pend = st;
            if (++st == p.nstages) { st = 0; ph ^= 1u; }
        }
        wg_wait<0>();
#pragma unroll
        for (int r = 0; r < WB_ACC_TAPS; ++r) wg_fence_acc(acc[r]);
        wg_fence_acc(accb);
    }

    // ================= partial sums straight from the fragments: (ci row, co pair) per register pair =================
    const int wr = (warp & 3) * 16 + (lane >> 2);       // fragment row (+8 for the second half)
    const int cc = 2 * (lane & 3);                      // fragment column (+8 j)
    const int taps = p.taps_total;
    if (rows_live) {
#pragma unroll
        for (int r = 0; r < WB_ACC_TAPS; ++r) {
            if (r >= p.kh) break;
            const int tap = p.tap0 + r * p.kw + s;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int ci_g = mb * 128 + mg * 64 + wr + 8 * h;
                if (ci_g >= p.ci) continue;
                float* prow = p.part + (((size_t)split * taps + tap) * p.ci + ci_g) * p.co;
#pragma unroll
                for (int j = 0; j < WB_BN / 8; ++j) {
                    const int co = nb * WB_BN + 8 * j + cc;
                    if (co < p.co)      // (co is a multiple of 4 and cc even: the pair is whole)
                        *reinterpret_cast<float2*>(prow + co) = make_float2(acc[r][4 * j + 2 * h], acc[r][4 * j + 2 * h + 1]);
                }
            }
        }
    }
    if (bias_here && (warp & 3) == 0 && (lane >> 2) == 0) {      // fragment row 0 holds sum_p dY[p][co]
#pragma unroll
        for (int j = 0; j < WB_BN / 8; ++j) {
            const int co = nb * WB_BN + 8 * j + cc;
            if (co < p.co) *reinterpret_cast<float2*>(p.bpart + (size_t)split * p.co + co) = make_float2(accb[4 * j], accb[4 * j + 1]);
        }
    }
}

// dw[i] = sum_k part[k][i] (fixed order), db[c] = sum_k bpart[k][c]
__global__ void wgrad_bf_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, size_t n4, int split,
                                       const float* __restrict__ bpart, float* __restrict__ db, int co, int accumulate,
                                       float wscale, float bscale) {
    pdl_prologue();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n4) {
        const float4* src = reinterpret_cast<const float4*>(part) + i;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = 0; k < split; ++k) {
            const float4 v = __ldcs(src + (size_t)k * n4);
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        a.x *= wscale; a.y *= wscale; a.z *= wscale; a.w *= wscale;      // undoes the 1/16 pre-scale of fp16 planes (exact)
        float4* d = reinterpret_cast<float4*>(dw) + i;
        if (accumulate) { const float4 o = *d; a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w; }
        *d = a;
    } else if (db && i < n4 + (size_t)co) {
        const int c = (int)(i - n4);
        float a = 0.f;
        for (int k = 0; k < split; ++k) a += bpart[(size_t)k * co + c];
        a *= bscale;
        if (accumulate) a += db[c];
        db[c] = a;
    }
}

struct WbPlan {
    int TH, nbox, box_rows, x_rows, nstages, nblocks, mblocks, xblk, splits, tiles_x, tiles_y, ntiles;
    uint32_t stage_bytes, x_plane_bytes, d_plane_bytes;
    bool ok;
};

static WbPlan wb_plan(const ConvWgrad& q) {
    WbPlan P{};
    const int ci = q.x.c, co = q.dy.c, kh = q.kh, kw = q.kw;
    P.ok = false;
    if (q.stride != 1 && q.stride != 2) return P;
    if (kh > WB_MAX_KH || kh * kw > 49) return P;
    if (ci < 3 || co < 16 || (co & 3)) return P;
    if ((size_t)q.dy.h * q.dy.w < 32) return P;
    P.nblocks = cdiv(co, WB_BN);
    P.mblocks = (ci + 127) / 128;
    P.xblk = ci > 64 ? 2 : 1;
    const size_t budget = 222 * 1024 - WB_ONES_BYTES;
    const int cand[4] = {16, 8, 4, 2};
    for (int i = 0; i < 4; ++i) {
        const int TH = cand[i];
        if (TH > 2 && TH >= 2 * q.dy.h) continue;                      // do not pad tiny maps to tall tiles
        const int halo = (kh - 1) * q.dil;
        const bool shared = q.stride == 1 && halo < (kh - 1) * TH && (TH + halo) <= 256;
        // stride 2, dilation 1: taps of equal row parity read the same strided patch (tap r = row r/2 of box r%2)
        const bool parity = q.stride == 2 && q.dil == 1 && kh > 2;
        const int nbox = shared ? 1 : (parity ? 2 : kh);
        const int box_rows = shared ? TH + halo : (parity ? TH + (kh - 1) / 2 : TH);
        const int x_rows = nbox * box_rows;
        const size_t xpb = (size_t)P.xblk * x_rows * WB_ATOM, dpb = (size_t)TH * WB_ATOM;
        const size_t stage = 2 * (xpb + dpb);
        const int ns = (int)std::min<size_t>(4, budget / stage);
        if (ns < 2 || (ns < 3 && TH > 2)) continue;
        if (box_rows * q.stride > 256) continue;
        P.TH = TH; P.nbox = nbox; P.box_rows = box_rows; P.x_rows = x_rows; P.nstages = ns;
        P.stage_bytes = (uint32_t)stage; P.x_plane_bytes = (uint32_t)xpb; P.d_plane_bytes = (uint32_t)dpb;
        P.ok = true;
        break;
    }
    if (!P.ok) return P;
    P.tiles_x = cdiv(q.dy.w, 8); P.tiles_y = cdiv(q.dy.h, P.TH);
    P.ntiles = q.dy.n * P.tiles_x * P.tiles_y;
    const int cols = kw * P.mblocks * P.nblocks;
    int splits = std::max(1, (NUM_SMS + cols / 2) / cols);
    splits = std::min(splits, std::min(P.ntiles, 64));
    // bound the number of accumulation steps per CTA (the tensor core adds into fp32 with truncation)
    const int max_tiles = std::max(1, 8192 / (8 * P.TH));
    splits = std::max(splits, std::min(64, cdiv(P.ntiles, max_tiles)));
    P.splits = std::max(1, std::min(splits, P.ntiles));
    return P;
}

bool wgrad_bf_supported(const ConvWgrad& q) { return wb_plan(q).ok; }

size_t wgrad_bf_workspace_floats(int kh, int kw, int ci, int co) {
    return 64 * ((size_t)kh * kw * ci * co + (size_t)co) + 64;
}

int wgrad_bf_init() {
    static bool done = false;
    if (done) return 0;
    MS_CHECK_CUDA(cudaFuncSetAttribute(wgrad_bf_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    MS_CHECK_CUDA(cudaFuncSetAttribute(wgrad_bf_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    done = true;
    return 0;
}

// One kernel launch over the filter rows [r0, r0 + q.kh) of a kh_total-row filter (q.pad_t already shifted to row r0).
// splits_force > 0: use that split factor (all row groups of one filter share the partial-sum layout).  Returns the split
// factor used through *splits_out.
static int wgrad_bf_launch(const ConvWgrad& q, const ActPlanes& xp, const ActPlanes& dp, int r0, int kh_total, int splits_force,
                           int* splits_out, cudaStream_t st) {
    WbPlan P = wb_plan(q);
    MS_REQUIRE(P.ok, "wgrad_bf: unsupported geometry");
    {   // the split factor never outgrows the caller's workspace
        const size_t per = (size_t)kh_total * q.kw * q.x.c * q.dy.c + (size_t)q.dy.c;
        P.splits = (int)std::max<size_t>(1, std::min<size_t>((size_t)P.splits, q.workspace_floats / std::max<size_t>(per, 1)));
        if (splits_force > 0) P.splits = std::max(1, std::min(splits_force, P.ntiles));
        MS_REQUIRE(splits_force <= 0 || P.splits == splits_force, "wgrad_bf: row groups disagree on the split factor");
    }
    MS_REQUIRE(xp.fmt == dp.fmt, "wgrad_bf: a wgmma takes one 16-bit element type; both plane sets must share a format");
    MS_REQUIRE(q.kh <= WB_ACC_TAPS, "wgrad_bf: more filter rows than accumulators in one launch");
    MS_REQUIRE(xp.hi && xp.lo && dp.hi && dp.lo && (xp.cs & 7) == 0 && (dp.cs & 7) == 0 && xp.cs >= q.x.c && dp.cs >= q.dy.c,
               "wgrad_bf: operand planes missing");
    if (wgrad_bf_init()) return -1;
    const int ci = q.x.c, co = q.dy.c, taps = kh_total * q.kw;
    const size_t wn = (size_t)taps * ci * co;
    MS_REQUIRE((wn & 3) == 0, "wgrad_bf: taps*ci*co must be a multiple of 4");
    MS_REQUIRE(q.workspace_floats >= wn + co, "wgrad_bf: workspace too small");
    MS_REQUIRE((reinterpret_cast<uintptr_t>(q.workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(q.dw) & 15) == 0,
               "wgrad_bf: workspace / dw must be 16-byte aligned");
    static WgradBfParams p;
    memset(&p, 0, sizeof p);
    p.kh = q.kh; p.kw = q.kw;
    p.tiles_x = P.tiles_x; p.tiles_y = P.tiles_y; p.ntiles = P.ntiles; p.splits = P.splits;
    p.TH = P.TH; p.sx = q.stride; p.nbox = P.nbox; p.box_rows = P.box_rows; p.x_rows = P.x_rows;
    const bool parity = q.stride == 2 && q.dil == 1 && q.kh > 2 && P.nbox == 2;
    for (int r = 0; r < q.kh; ++r) {
        if (P.nbox == 1) { p.tap_row[r] = (short)(r * q.dil); }
        else if (parity) { p.tap_row[r] = (short)((r & 1) * P.box_rows + (r >> 1)); }
        else { p.tap_row[r] = (short)(r * P.TH); p.box_dy[r] = (short)(r * q.dil - q.pad_t); }
    }
    if (P.nbox == 1) p.box_dy[0] = (short)(-q.pad_t);
    if (parity) { p.box_dy[0] = (short)(-q.pad_t); p.box_dy[1] = (short)(1 - q.pad_t); }
    p.pad_l = q.pad_l; p.dil = q.dil;
    p.ci = ci; p.co = co; p.mblocks = P.mblocks; p.nblocks = P.nblocks; p.xblk = P.xblk;
    p.nstages = P.nstages; p.stage_bytes = P.stage_bytes; p.x_plane_bytes = P.x_plane_bytes; p.d_plane_bytes = P.d_plane_bytes;
    p.with_bias = (q.db && r0 == 0) ? 1 : 0;
    p.tap0 = r0 * q.kw; p.taps_total = taps;
    p.part = q.workspace;
    p.bpart = q.workspace + (size_t)P.splits * wn;

    const CUtensorMap *mXh, *mXl, *mDh, *mDl;
    {
        cuuint64_t dims[4] = {(cuuint64_t)ci, (cuuint64_t)q.x.w, (cuuint64_t)q.x.h, (cuuint64_t)q.x.n};
        cuuint64_t strides[3] = {(cuuint64_t)xp.cs * 2, (cuuint64_t)q.x.w * xp.cs * 2, (cuuint64_t)q.x.h * q.x.w * xp.cs * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)(8 * q.stride), (cuuint32_t)(P.box_rows * q.stride), 1};
        cuuint32_t es[4] = {1, (cuuint32_t)q.stride, (cuuint32_t)q.stride, 1};
        if (bf_get_map(&mXh, xp.hi, 4, dims, strides, box, es, 128)) return -1;
        if (bf_get_map(&mXl, xp.lo, 4, dims, strides, box, es, 128)) return -1;
    }
    {
        cuuint64_t dims[4] = {(cuuint64_t)co, (cuuint64_t)q.dy.w, (cuuint64_t)q.dy.h, (cuuint64_t)q.dy.n};
        cuuint64_t strides[3] = {(cuuint64_t)dp.cs * 2, (cuuint64_t)q.dy.w * dp.cs * 2, (cuuint64_t)q.dy.h * q.dy.w * dp.cs * 2};
        cuuint32_t box[4] = {64, 8, (cuuint32_t)P.TH, 1};
        cuuint32_t es[4] = {1, 1, 1, 1};
        if (bf_get_map(&mDh, dp.hi, 4, dims, strides, box, es, 128)) return -1;
        if (bf_get_map(&mDl, dp.lo, 4, dims, strides, box, es, 128)) return -1;
    }
    const size_t smem = WB_ONES_BYTES + (size_t)P.nstages * P.stage_bytes + 1024;
    const dim3 grid(q.kw * P.mblocks * P.nblocks, P.splits);
    launch_k(xp.fmt == 0 ? wgrad_bf_kernel<1> : wgrad_bf_kernel<0>, grid, dim3(WB_THREADS), smem, st, *mXh, *mXl, *mDh, *mDl, p);
    if (splits_out) *splits_out = P.splits;
    return check_launch("wgrad_bf");
}

// Filter rows per launch.  Every filter row keeps its own register accumulator (WB_BN / 2 floats per thread, plus the bias
// accumulator), so filters with more than WB_ACC_TAPS rows run as groups of at most that many rows, each group its own
// launch with its own, shorter halo.
static int wb_group_rows(const ConvWgrad& q) { return std::min(q.kh, WB_ACC_TAPS); }

// xp / dp: bf16 planes of q.x / q.dy
int wgrad_bf(const ConvWgrad& q, const ActPlanes& xp, const ActPlanes& dp, cudaStream_t st) {
    const int khg = wb_group_rows(q);
    int splits = 0;
    for (int r0 = 0; r0 < q.kh; r0 += khg) {
        ConvWgrad g = q;
        g.kh = std::min(khg, q.kh - r0);
        g.pad_t = q.pad_t - r0 * q.dil;
        if (r0) g.db = q.db;                       // (bias only in the first group; the launch looks at r0)
        MS_REQUIRE(wb_plan(g).ok, "wgrad_bf: unsupported geometry");
        if (r0 == 0 && khg < q.kh) {               // the shortest group has the same tile count: plans agree on ntiles, take the first group's split
            WbPlan P0 = wb_plan(g);
            const size_t per = (size_t)q.kh * q.kw * q.x.c * q.dy.c + (size_t)q.dy.c;
            splits = (int)std::max<size_t>(1, std::min<size_t>((size_t)P0.splits, q.workspace_floats / std::max<size_t>(per, 1)));
            for (int r1 = khg; r1 < q.kh; r1 += khg) {      // ... clamped to what every group can honour
                ConvWgrad h = q; h.kh = std::min(khg, q.kh - r1); h.pad_t = q.pad_t - r1 * q.dil;
                WbPlan P1 = wb_plan(h);
                MS_REQUIRE(P1.ok, "wgrad_bf: unsupported geometry");
                splits = std::min(splits, P1.ntiles);
            }
            splits = std::min(splits, P0.ntiles);
        }
        int used = 0;
        if (wgrad_bf_launch(g, xp, dp, r0, q.kh, splits, &used, st)) return -1;
        splits = used;
    }
    const int ci = q.x.c, co = q.dy.c, taps = q.kh * q.kw;
    const size_t wn = (size_t)taps * ci * co;
    float* part = q.workspace;
    float* bpart = q.workspace + (size_t)splits * wn;
    struct { int splits; } P{splits};
    struct { float* part; float* bpart; } p{part, bpart};
    const size_t n4 = wn / 4;
    const size_t work = n4 + (q.db ? (size_t)co : 0);
    const float sx16 = xp.fmt == 1 ? 1.f / xp.scale : 1.f, sd16 = dp.fmt == 1 ? 1.f / dp.scale : 1.f;
    launch_k(wgrad_bf_reduce_kernel, dim3((unsigned)cdivz(work, 256)), dim3(256), 0, st, p.part, q.dw, n4, P.splits, p.bpart, q.db, co, q.accumulate,
                                                                      sx16 * sd16, sd16);
    return check_launch("wgrad_bf_reduce", 1);
}

// one-shot convenience (operator-level C ABI / tests): splits x and dy into planes, runs the kernel.
//   scratch layout (bytes): [x hi | x lo | dy hi | dy lo | partial sums]
size_t wgrad_bf_oneshot_scratch_bytes(const ConvWgrad& q) {
    const size_t xe = q.x.pixels() * ((q.x.c + 7) / 8 * 8), de = q.dy.pixels() * ((q.dy.c + 7) / 8 * 8);
    return 2 * (xe * 2 + 256) + 2 * (de * 2 + 256) + wgrad_bf_workspace_floats(q.kh, q.kw, q.x.c, q.dy.c) * 4 + 1024;
}

int wgrad_bf_oneshot(const ConvWgrad& q0, void* scratch, size_t scratch_bytes, cudaStream_t st) {
    MS_REQUIRE(wgrad_bf_supported(q0), "wgrad_bf: unsupported geometry");
    MS_REQUIRE(scratch_bytes >= wgrad_bf_oneshot_scratch_bytes(q0), "wgrad_bf: scratch too small");
    MS_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, "wgrad_bf: scratch must be 256B aligned");
    unsigned char* b = reinterpret_cast<unsigned char*>(scratch);
    auto take = [&](size_t bytes) { unsigned char* r = b; b += (bytes + 255) / 256 * 256; return r; };
    ActPlanes xp, dp;
    xp.cs = (q0.x.c + 7) / 8 * 8; dp.cs = (q0.dy.c + 7) / 8 * 8; xp.fmt = 0; dp.fmt = 0; xp.scale = dp.scale = 1.f;
    const size_t xe = q0.x.pixels() * xp.cs, de = q0.dy.pixels() * dp.cs;
    xp.hi = take(xe * 2); xp.lo = take(xe * 2); dp.hi = take(de * 2); dp.lo = take(de * 2);
    ConvWgrad q = q0;
    q.workspace_floats = wgrad_bf_workspace_floats(q.kh, q.kw, q.x.c, q.dy.c);
    q.workspace = reinterpret_cast<float*>(take(q.workspace_floats * 4));
    if (split_planes(q.x, xp, st)) return -1;
    if (split_planes(q.dy, dp, st)) return -1;
    return wgrad_bf(q, xp, dp, st);
}

}  // namespace ms
