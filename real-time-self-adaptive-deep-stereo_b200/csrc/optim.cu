// Momentum-SGD update over a contiguous parameter / gradient / momentum arena.
// Replaces tf.train.MomentumOptimizer(lr, 0.9) ApplyMomentum ops (reference Stereo_Online_Adaptation.py:85,
// :118, :128): accum = mu*accum + g ; var -= lr*accum (non-Nesterov).  `gscale` folds the 1/N of the
// data-parallel gradient mean into the same pass (the all-reduce delivers the sum).
#include "common.cuh"

namespace ms {

__global__ void momentum_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m, size_t n,
                                float lr, float mu, float gscale) {
    pdl_prologue();
    size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        float4 gv = *reinterpret_cast<const float4*>(g + i);
        float4 mv = *reinterpret_cast<float4*>(m + i);
        float4 wv = *reinterpret_cast<float4*>(w + i);
        mv.x = mu * mv.x + gv.x * gscale; mv.y = mu * mv.y + gv.y * gscale;
        mv.z = mu * mv.z + gv.z * gscale; mv.w = mu * mv.w + gv.w * gscale;
        wv.x -= lr * mv.x; wv.y -= lr * mv.y; wv.z -= lr * mv.z; wv.w -= lr * mv.w;
        *reinterpret_cast<float4*>(m + i) = mv;
        *reinterpret_cast<float4*>(w + i) = wv;
    } else {
        for (; i < n; ++i) {
            float mv = mu * m[i] + g[i] * gscale;
            m[i] = mv;
            w[i] -= lr * mv;
        }
    }
}

int momentum_update(float* w, const float* g, float* m, size_t n, float lr, float mu, float gscale, cudaStream_t st) {
    if (n == 0) return 0;
    MS_REQUIRE(((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m)) & 15) == 0,
               "momentum_update: arenas must be 16B aligned");
    size_t nthr = cdivz(n, 4);
    launch_k(momentum_kernel, dim3((unsigned)cdivz(nthr, 256)), dim3(256), 0, st, w, g, m, n, lr, mu, gscale);
    return check_launch("momentum_update");
}

// Adam update.  Replaces tf.train.AdamOptimizer(lr) (reference Demo/demo_model.py:163) as its ApplyAdam kernel applies it:
//   lr_t = lr * sqrt(1 - beta2_power) / (1 - beta1_power)
//   m += (g - m) * (1 - beta1) ;  v += (g*g - v) * (1 - beta2) ;  w -= lr_t * m / (eps + sqrt(v))
// The powers are the optimizer's one pair of non-slot variables (shared by every train op): every block reads them from
// device memory, and a second launch advances them only after the whole update has completed (PDL waits for it).
__device__ __forceinline__ void adam_one(float& w, float g, float& m, float& v, float lr_t, float b1, float b2, float eps) {
    m += (g - m) * (1.f - b1);
    v += (g * g - v) * (1.f - b2);
    w -= lr_t * m / (eps + sqrtf(v));
}

__global__ void adam_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            const float* __restrict__ powers, size_t n, float lr, float b1, float b2, float eps, float gscale) {
    pdl_prologue();
    const float lr_t = lr * sqrtf(1.f - powers[1]) / (1.f - powers[0]);
    size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        float4 gv = *reinterpret_cast<const float4*>(g + i);
        float4 mv = *reinterpret_cast<float4*>(m + i);
        float4 vv = *reinterpret_cast<float4*>(v + i);
        float4 wv = *reinterpret_cast<float4*>(w + i);
        adam_one(wv.x, gv.x * gscale, mv.x, vv.x, lr_t, b1, b2, eps);
        adam_one(wv.y, gv.y * gscale, mv.y, vv.y, lr_t, b1, b2, eps);
        adam_one(wv.z, gv.z * gscale, mv.z, vv.z, lr_t, b1, b2, eps);
        adam_one(wv.w, gv.w * gscale, mv.w, vv.w, lr_t, b1, b2, eps);
        *reinterpret_cast<float4*>(m + i) = mv;
        *reinterpret_cast<float4*>(v + i) = vv;
        *reinterpret_cast<float4*>(w + i) = wv;
    } else {
        for (; i < n; ++i) adam_one(w[i], g[i] * gscale, m[i], v[i], lr_t, b1, b2, eps);
    }
}

__global__ void adam_powers_kernel(float* powers, float b1, float b2) {
    pdl_prologue();
    powers[0] *= b1;
    powers[1] *= b2;
}

int adam_update(float* w, const float* g, float* m, float* v, float* powers, size_t n, float lr, float b1, float b2, float eps,
                float gscale, cudaStream_t st) {
    MS_REQUIRE(powers != nullptr, "adam_update: no beta powers");
    MS_REQUIRE(((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                 reinterpret_cast<uintptr_t>(v)) & 15) == 0, "adam_update: arenas must be 16B aligned");
    if (n > 0) {
        size_t nthr = cdivz(n, 4);
        launch_k(adam_kernel, dim3((unsigned)cdivz(nthr, 256)), dim3(256), 0, st, w, g, m, v, (const float*)powers, n, lr, b1,
                 b2, eps, gscale);
    }
    launch_k(adam_powers_kernel, dim3(1), dim3(1), 0, st, powers, b1, b2);
    return check_launch("adam_update", n > 0 ? 2 : 1);
}

}  // namespace ms
