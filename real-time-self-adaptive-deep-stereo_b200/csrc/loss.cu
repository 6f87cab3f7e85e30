// Reprojection loss  L = 0.85*mean(clip((1-SSIM)/2,0,1)) + 0.15*mean|warp(right,D) - left|  and dL/dD.
//
// Replaces loss_factory.get_reprojection_loss('mean_SSIM_l1') (reference Losses/loss_factory.py:353-395),
// mean_SSIM_L1/mean_SSIM/SSIM/mean_l1 (:28-38,:128-164) and preprocessing.warp_image/bilinear_sampler
// (Data_utils/preprocessing.py:121-230) plus the backward sub-graph tf.gradients derives from them.
// Images are divided by 256 (loss_factory.py:373-374); the sampler clamps indices and does NOT mask the
// weights (preprocessing.py:159-167); the SSIM pools are 3x3 VALID (loss_factory.py:137-142).
//
// Three HBM-bound passes over full-resolution maps + a fixed-order (deterministic) fp64 final reduction.
#include "common.cuh"

namespace ms {

constexpr int LB = 256;

__device__ __forceinline__ float block_sum(float v, float* sm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) sm[wid] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 32) {
        t = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

// pass A: warped image, d(warped)/dD, L1 partial sums
__global__ void __launch_bounds__(LB) loss_warp_kernel(ReprojLoss p, float* __restrict__ xw, float* __restrict__ dxw,
                                                       float* __restrict__ l1_partial) {
    pdl_prologue();
    __shared__ float sm[32];
    const size_t total = (size_t)p.B * p.H * p.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    float l1 = 0.f;
    if (i < total) {
        const int x = (int)(i % p.W);
        const size_t rowbase = i - x;
        const float cx = (float)x - p.disp[i];
        const float x0 = floorf(cx), x1 = x0 + 1.f;
        const float w0 = x1 - cx, w1 = cx - x0;
        const int i0 = (int)fminf(fmaxf(x0, 0.f), (float)(p.W - 1));
        const int i1 = (int)fminf(fmaxf(x1, 0.f), (float)(p.W - 1));
        const float* r0 = p.right + (rowbase + i0) * 3;
        const float* r1 = p.right + (rowbase + i1) * 3;
        const float* l = p.left + i * 3;
        const float s = 1.f / 256.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float a = r0[c] * s, b = r1[c] * s;
            float v = w0 * a + w1 * b;
            xw[i * 3 + c] = v;
            dxw[i * 3 + c] = a - b;          // d v / d D  (cx = x - D)
            l1 += fabsf(v - l[c] * s);
        }
    }
    float t = block_sum(l1, sm);
    if (threadIdx.x == 0) l1_partial[blockIdx.x] = t;
}

// pass B: one thread per 3x3 window centre (VALID): SSIM term + derivative coefficients
__global__ void __launch_bounds__(LB) loss_ssim_kernel(ReprojLoss p, const float* __restrict__ xw,
                                                       float* __restrict__ coef, float* __restrict__ ss_partial,
                                                       float gwin) {
    pdl_prologue();
    __shared__ float sm[32];
    const int WH = p.H - 2, WW = p.W - 2;
    const size_t total = (size_t)p.B * WH * WW;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    float ssum = 0.f;
    if (i < total) {
        const int wx = (int)(i % WW);
        const size_t q = i / WW;
        const int wy = (int)(q % WH);
        const int b = (int)(q / WH);
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float s = 1.f / 256.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float sx = 0.f, sy = 0.f, sxx = 0.f, syy = 0.f, sxy = 0.f;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    size_t pi = ((size_t)(b * p.H + wy + dy) * p.W + wx + dx) * 3 + c;
                    float xv = xw[pi], yv = p.left[pi] * s;
                    sx += xv; sy += yv; sxx += xv * xv; syy += yv * yv; sxy += xv * yv;
                }
            const float mx = sx / 9.f, my = sy / 9.f;
            const float vx = sxx / 9.f - mx * mx, vy = syy / 9.f - my * my, vxy = sxy / 9.f - mx * my;
            const float n1 = 2.f * mx * my + C1, n2 = 2.f * vxy + C2;
            const float d1 = mx * mx + my * my + C1, d2 = vx + vy + C2;
            const float S = (n1 * n2) / (d1 * d2);
            const float f = (1.f - S) * 0.5f;
            ssum += fminf(fmaxf(f, 0.f), 1.f);
            if (coef) {
                float g = (f >= 0.f && f <= 1.f) ? (-0.5f * gwin) : 0.f;   // d loss / d S
                const float dd = d1 * d2;
                // partials of S holding E[x^2], E[xy] fixed
                const float dS_dmx = ((2.f * my * n2 - 2.f * my * n1) * dd - n1 * n2 * (2.f * mx * d2 - 2.f * mx * d1)) / (dd * dd);
                const float dS_dExx = -(n1 * n2) * d1 / (dd * dd);
                const float dS_dExy = 2.f * n1 / dd;
                float* o = coef + (i * 3 + c) * 3;
                o[0] = g * dS_dmx / 9.f;
                o[1] = g * dS_dExx * 2.f / 9.f;
                o[2] = g * dS_dExy / 9.f;
            }
        }
    }
    float t = block_sum(ssum, sm);
    if (threadIdx.x == 0) ss_partial[blockIdx.x] = t;
}

// pass C: per pixel gather of the <=9 windows covering it, + L1 term, chain through the warp
__global__ void __launch_bounds__(LB) loss_grad_kernel(ReprojLoss p, const float* __restrict__ xw,
                                                       const float* __restrict__ dxw, const float* __restrict__ coef,
                                                       float gl1) {
    pdl_prologue();
    const size_t total = (size_t)p.B * p.H * p.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int x = (int)(i % p.W);
    const size_t q = i / p.W;
    const int y = (int)(q % p.H);
    const int b = (int)(q / p.H);
    const int WH = p.H - 2, WW = p.W - 2;
    const float s = 1.f / 256.f;
    float a[3] = {0.f, 0.f, 0.f}, bq[3] = {0.f, 0.f, 0.f}, cq[3] = {0.f, 0.f, 0.f};
    for (int wy = max(0, y - 2); wy <= min(WH - 1, y); ++wy)
        for (int wx = max(0, x - 2); wx <= min(WW - 1, x); ++wx) {
            const float* o = coef + (((size_t)(b * WH + wy) * WW + wx) * 3) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) { a[c] += o[c * 3]; bq[c] += o[c * 3 + 1]; cq[c] += o[c * 3 + 2]; }
        }
    float g = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float xv = xw[i * 3 + c], yv = p.left[i * 3 + c] * s;
        float gx = a[c] + bq[c] * xv + cq[c] * yv;
        const float df = xv - yv;
        gx += gl1 * (df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f));
        g += gx * dxw[i * 3 + c];
    }
    p.ddisp[i] = g * p.grad_scale;
}

__global__ void loss_final_kernel(const float* __restrict__ l1_partial, int n1, const float* __restrict__ ss_partial,
                                  int n2, double inv_np, double inv_nw, float* __restrict__ loss) {
    pdl_prologue();
    __shared__ double sm1[256], sm2[256];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < n1; i += 256) a += (double)l1_partial[i];
    for (int i = threadIdx.x; i < n2; i += 256) b += (double)ss_partial[i];
    sm1[threadIdx.x] = a; sm2[threadIdx.x] = b;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { sm1[threadIdx.x] += sm1[threadIdx.x + o]; sm2[threadIdx.x] += sm2[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss = (float)(0.85 * sm2[0] * inv_nw + 0.15 * sm1[0] * inv_np);
}

// workspace layout: [xw 3n | dxw 3n | L1 partials | SSIM partials | coef 9n]; the gradient coefficients come last so that
// a pass without gradient needs only loss_value_workspace_floats
size_t loss_value_workspace_floats(int B, int H, int W) {
    size_t n = (size_t)B * H * W;
    return n * 3 * 2 + 2 * (n / LB + 2) + 64;
}
size_t loss_workspace_floats(int B, int H, int W) { return loss_value_workspace_floats(B, H, W) + (size_t)B * H * W * 9; }

int reproj_loss(const ReprojLoss& p, cudaStream_t st) {
    MS_REQUIRE(p.H >= 3 && p.W >= 3, "reproj_loss: image too small for 3x3 SSIM windows");
    const size_t n = (size_t)p.B * p.H * p.W;
    const size_t nwin = (size_t)p.B * (p.H - 2) * (p.W - 2);
    float* xw = p.workspace;
    float* dxw = xw + n * 3;
    float* l1p = dxw + n * 3;
    const int nb1 = (int)cdivz(n, LB), nb2 = (int)cdivz(nwin, LB);
    float* ssp = l1p + nb1 + 1;
    float* coef = ssp + nb2 + 1;
    const double inv_np = 1.0 / ((double)n * 3.0), inv_nw = 1.0 / ((double)nwin * 3.0);
    launch_k(loss_warp_kernel, dim3(nb1), dim3(LB), 0, st, p, xw, dxw, l1p);
    launch_k(loss_ssim_kernel, dim3(nb2), dim3(LB), 0, st, p, xw, p.ddisp ? coef : nullptr, ssp, (float)(0.85 * inv_nw));
    if (p.ddisp) launch_k(loss_grad_kernel, dim3(nb1), dim3(LB), 0, st, p, xw, dxw, coef, (float)(0.15 * inv_np));
    launch_k(loss_final_kernel, dim3(1), dim3(256), 0, st, l1p, nb1, ssp, nb2, inv_np, inv_nw, p.loss);
    return check_launch("reproj_loss", p.ddisp ? 4 : 3);
}

// ---------------------------------------------------------------------------------------------------------------------
// Proxy-label loss of the continual-adaptation variant (reference Losses/loss_factory.py:304-351 `get_proxy_loss('mean_l1')`,
// :28-38 `mean_l1`; used by Stereo_Continual_Adaptation.py:75,112):
//     valid = !(proxy <= 0 || proxy >= 192);   loss = weight * sum(valid * |d - proxy|) / sum(valid)
// (prediction already at the proxy's resolution: `resize_to_prediction` is the identity on this path, scale factor 1).
// Three small kernels: per-block partial sums (fixed order), one fp64 final sum that also leaves 1 / sum(valid) for the
// gradient pass, and d loss / d d = weight * valid * sign(d - proxy) / sum(valid).  An image without a single valid proxy
// pixel gives 0 / 0 = NaN in the reference; here the loss and its gradient are 0 (documented difference).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void proxy_partial_kernel(const float* __restrict__ disp, const float* __restrict__ proxy, int n, float* __restrict__ part) {
    pdl_prologue();
    __shared__ float sm[32];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float e = 0.f, v = 0.f;
    if (i < n) {
        const float p = proxy[i];
        if (!(p <= 0.f || p >= 192.f)) { v = 1.f; e = fabsf(disp[i] - p); }
    }
    const float te = block_sum(e, sm);
    const float tv = block_sum(v, sm);
    if (threadIdx.x == 0) { part[blockIdx.x * 2] = te; part[blockIdx.x * 2 + 1] = tv; }
}
__global__ void proxy_final_kernel(const float* __restrict__ part, int nb, float weight, float* __restrict__ loss, float* __restrict__ inv_count) {
    pdl_prologue();
    __shared__ double s[2][256];
    double a = 0, b = 0;
    for (int i = threadIdx.x; i < nb; i += 256) { a += part[i * 2]; b += part[i * 2 + 1]; }
    s[0][threadIdx.x] = a; s[1][threadIdx.x] = b;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { s[0][threadIdx.x] += s[0][threadIdx.x + o]; s[1][threadIdx.x] += s[1][threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double cnt = s[1][0];
        *loss = cnt > 0.0 ? (float)((double)weight * s[0][0] / cnt) : 0.f;
        *inv_count = cnt > 0.0 ? (float)(1.0 / cnt) : 0.f;
    }
}
__global__ void proxy_grad_kernel(const float* __restrict__ disp, const float* __restrict__ proxy, int n, float scale,
                                  const float* __restrict__ inv_count, float* __restrict__ ddisp) {
    pdl_prologue();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float p = proxy[i];
    float g = 0.f;
    if (!(p <= 0.f || p >= 192.f)) {
        const float d = disp[i] - p;
        g = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * scale * __ldg(inv_count);      // tf.abs' gradient is sign(x): 0 at 0
    }
    ddisp[i] = g;
}
// workspace: >= 2 * ceil(n / 256) + 2 floats
int proxy_loss(const float* disp, const float* proxy, int n, float weight, float grad_scale, float* loss, float* ddisp,
               float* workspace, cudaStream_t st) {
    const int nb = cdiv(n, LB);
    float* inv_count = workspace + (size_t)nb * 2;
    launch_k(proxy_partial_kernel, dim3(nb), dim3(LB), 0, st, disp, proxy, n, workspace);
    launch_k(proxy_final_kernel, dim3(1), dim3(256), 0, st, workspace, nb, weight, loss, inv_count);
    if (ddisp) launch_k(proxy_grad_kernel, dim3(nb), dim3(LB), 0, st, disp, proxy, n, weight * grad_scale, inv_count, ddisp);
    return check_launch("proxy_loss", ddisp ? 3 : 2);
}

// EPE / bad3 against ground truth (reference Stereo_Online_Adaptation.py:74-82); out2 = {epe, bad3}
__global__ void epe_partial_kernel(const float* __restrict__ disp, const float* __restrict__ gt, int n,
                                   float* __restrict__ part) {
    pdl_prologue();
    __shared__ float sm[32];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    float e = 0.f, v = 0.f, bad = 0.f;
    if (i < n) {
        float g = gt[i];
        if (g != 0.f) { v = 1.f; e = fabsf(disp[i] - g); bad = e > 3.f ? 1.f : 0.f; }
    }
    float te = block_sum(e, sm);
    float tv = block_sum(v, sm);
    float tb = block_sum(bad, sm);
    if (threadIdx.x == 0) { part[blockIdx.x * 3] = te; part[blockIdx.x * 3 + 1] = tv; part[blockIdx.x * 3 + 2] = tb; }
}
__global__ void epe_final_kernel(const float* __restrict__ part, int nb, float* __restrict__ out2) {
    pdl_prologue();
    __shared__ double s[3][256];
    double a = 0, b = 0, c = 0;
    for (int i = threadIdx.x; i < nb; i += 256) { a += part[i * 3]; b += part[i * 3 + 1]; c += part[i * 3 + 2]; }
    s[0][threadIdx.x] = a; s[1][threadIdx.x] = b; s[2][threadIdx.x] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) for (int k = 0; k < 3; ++k) s[k][threadIdx.x] += s[k][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) { out2[0] = (float)(s[0][0] / s[1][0]); out2[1] = (float)(s[2][0] / s[1][0]); }
}
int epe_bad3(const float* disp, const float* gt, int n, float* out2, float* workspace, cudaStream_t st) {
    int nb = cdiv(n, LB);
    launch_k(epe_partial_kernel, dim3(nb), dim3(LB), 0, st, disp, gt, n, workspace);
    launch_k(epe_final_kernel, dim3(1), dim3(256), 0, st, workspace, nb, out2);
    return check_launch("epe_bad3", 2);
}

}  // namespace ms
