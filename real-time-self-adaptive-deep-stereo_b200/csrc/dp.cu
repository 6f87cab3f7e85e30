// Data-parallel gradient exchange fused with the optimizer: ONE kernel per step does the all-reduce of the adapted
// module's gradient range over NVLink peer memory AND the momentum update (new functionality, SURVEY 8e: the reference
// is single-GPU; N ranks with one frame each equal its graph at batch N because every loss is a batch mean,
// Losses/loss_factory.py:38,160).
//
// Each rank owns an exchange buffer (cudaMalloc, IPC-mapped into every peer):  [gradient range | loss scalars].
//   dp_pack_kernel          copies the module's gradient range and the two loss scalars into the local buffer
//                           (after all peers finished reading the previous step's content).
//   dp_reduce_update_kernel signals "ready" into every peer's flag array, waits for every peer's "ready" in its OWN
//                           flag array (local polling, acquire at system scope), then every rank reads the SAME
//                           N buffers in the SAME rank order (one-shot all-reduce: (N-1) x payload <= 32 MB over
//                           NVSwitch per rank, bitwise identical sums everywhere), applies
//                               m = mu*m + g_sum/N ;  w -= lr*m
//                           to its own replica, stores the summed gradient, writes the mean losses, and finally signals
//                           "done" so the peers may overwrite their buffers in the next step.
// Flags carry the step epoch (never reset) and the module id: ranks that disagree about the module being adapted are
// detected instead of silently mixing gradients.  Every spin loop has a wall-clock timeout: a lost peer makes the
// step fail (NaN loss -> host error), never hang the GPU.  Both kernels are captured into the step's CUDA graph.
#include <cuda.h>

#include "common.cuh"
#include "engine.h"

namespace ms {

constexpr unsigned long long DP_TIMEOUT_NS = 30ull * 1000ull * 1000ull * 1000ull;

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_volatile4(const float* p) {
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

struct DpPeers {
    const float* xbuf[DP_MAX_WORLD];
    DpState* state[DP_MAX_WORLD];
};

// one block per ~4K floats; thread t < world polls the `done` flag of peer t
__global__ void dp_pack_kernel(DpState* __restrict__ st, int world, int rank, const float* __restrict__ g, size_t n,
                               const float* __restrict__ scalars, float* __restrict__ xbuf) {
    __shared__ unsigned int s_epoch;
    if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned int*>(&st->epoch);
    __syncthreads();
    const unsigned int e = s_epoch;
    if ((int)threadIdx.x < world && (int)threadIdx.x != rank) {
        const unsigned long long t0 = global_ns();
        while (ld_acquire_sys(&st->done[threadIdx.x]) + 1u < e) {
            if (global_ns() - t0 > DP_TIMEOUT_NS) { atomicExch(&st->error, 1u); break; }
            __nanosleep(64);
        }
    }
    __syncthreads();
    const size_t n4 = n >> 2;
    const float4* src = reinterpret_cast<const float4*>(g);
    float4* dst = reinterpret_cast<float4*>(xbuf);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
    if (blockIdx.x == 0 && threadIdx.x < 4) xbuf[n + threadIdx.x] = scalars[threadIdx.x];
}

__global__ void dp_reduce_update_kernel(DpState* __restrict__ st, const __grid_constant__ DpPeers peers, int world, int rank,
                                        unsigned int tag, size_t n, float* __restrict__ w, float* __restrict__ g,
                                        float* __restrict__ m, float lr, float mu, float gscale, float* __restrict__ scalars) {
    __shared__ unsigned int s_epoch;
    if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned int*>(&st->epoch);
    __syncthreads();
    const unsigned int e = s_epoch;
    const unsigned int token = (e << 8) | (tag & 0xffu);
    if (blockIdx.x == 0 && (int)threadIdx.x < world && (int)threadIdx.x != rank) {
        __threadfence_system();
        st_release_sys(&peers.state[threadIdx.x]->ready[rank], token);
    }
    if ((int)threadIdx.x < world && (int)threadIdx.x != rank) {
        const unsigned long long t0 = global_ns();
        unsigned int v;
        while (((v = ld_acquire_sys(&st->ready[threadIdx.x])) >> 8) < e) {
            if (global_ns() - t0 > DP_TIMEOUT_NS) { atomicExch(&st->error, 1u); break; }
            __nanosleep(32);
        }
        if ((v >> 8) == e && (v & 0xffu) != (tag & 0xffu)) atomicExch(&st->error, 2u);
    }
    __syncthreads();

    const size_t n4 = n >> 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < world; ++r) {               // fixed order on every rank: identical sums everywhere
            const float4 v = ld_volatile4(peers.xbuf[r] + 4 * i);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        float4 mv = reinterpret_cast<float4*>(m)[i];
        float4 wv = reinterpret_cast<float4*>(w)[i];
        mv.x = mu * mv.x + s.x * gscale; mv.y = mu * mv.y + s.y * gscale;
        mv.z = mu * mv.z + s.z * gscale; mv.w = mu * mv.w + s.w * gscale;
        wv.x -= lr * mv.x; wv.y -= lr * mv.y; wv.z -= lr * mv.z; wv.w -= lr * mv.w;
        reinterpret_cast<float4*>(m)[i] = mv;
        reinterpret_cast<float4*>(w)[i] = wv;
        reinterpret_cast<float4*>(g)[i] = s;
    }
    if (blockIdx.x == 0 && threadIdx.x < 2) {           // mean full-resolution loss / module loss over the ranks
        float s = 0.f;
        for (int r = 0; r < world; ++r) s += *reinterpret_cast<const volatile float*>(peers.xbuf[r] + n + threadIdx.x);
        s *= gscale;
        if (*reinterpret_cast<volatile unsigned int*>(&st->error) != 0u) s = __int_as_float(0x7fc00000);
        scalars[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(&st->blocks_done, 1u);
        if (old == gridDim.x - 1) {
            st->blocks_done = 0u;
            st->epoch = e + 1u;
            __threadfence_system();
            for (int r = 0; r < world; ++r)
                if (r != rank) st_release_sys(&peers.state[r]->done[rank], e);
        }
    }
}

int Engine::dp_create(int rank, int world, unsigned char* handles_out) {
    MS_REQUIRE(world >= 2 && world <= DP_MAX_WORLD && rank >= 0 && rank < world, "dp_create: bad rank / world size");
    MS_REQUIRE(bound, "dp_create: engine not bound");
    MS_REQUIRE(!dp_xbuf, "dp_create: already created");
    dp_cap_floats = n_params + 64;
    void *xb = nullptr, *stt = nullptr;
    MS_CHECK_CUDA(cudaMalloc(&xb, dp_cap_floats * sizeof(float)));
    MS_CHECK_CUDA(cudaMalloc(&stt, sizeof(DpState)));
    MS_CHECK_CUDA(cudaMemset(xb, 0, dp_cap_floats * sizeof(float)));
    DpState init;
    memset(&init, 0, sizeof init);
    init.epoch = 1u;
    MS_CHECK_CUDA(cudaMemcpy(stt, &init, sizeof init, cudaMemcpyHostToDevice));
    dp_xbuf = static_cast<float*>(xb); dp_state = static_cast<DpState*>(stt);
    dp_rank = rank; dp_world = world;
    cudaIpcMemHandle_t hx, hs;
    MS_CHECK_CUDA(cudaIpcGetMemHandle(&hx, xb));
    MS_CHECK_CUDA(cudaIpcGetMemHandle(&hs, stt));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(handles_out, &hx, 64);
    memcpy(handles_out + 64, &hs, 64);
    return 0;
}

int Engine::dp_connect(const unsigned char* all_handles) {
    MS_REQUIRE(dp_xbuf && dp_state, "dp_connect: dp_create first");
    for (int r = 0; r < dp_world; ++r) {
        if (r == dp_rank) { dp_peer_xbuf[r] = dp_xbuf; dp_peer_state[r] = dp_state; continue; }
        cudaIpcMemHandle_t hx, hs;
        memcpy(&hx, all_handles + (size_t)r * 128, 64);
        memcpy(&hs, all_handles + (size_t)r * 128 + 64, 64);
        void *px = nullptr, *ps = nullptr;
        MS_CHECK_CUDA(cudaIpcOpenMemHandle(&px, hx, cudaIpcMemLazyEnablePeerAccess));
        MS_CHECK_CUDA(cudaIpcOpenMemHandle(&ps, hs, cudaIpcMemLazyEnablePeerAccess));
        dp_peer_xbuf[r] = static_cast<float*>(px); dp_peer_state[r] = static_cast<DpState*>(ps);
    }
    dp_connected = true;
    return 0;
}

// all-reduce of the group's gradient range + loss scalars fused with the momentum update (gscale = 1/world)
int Engine::dp_update(int group, float lr, float mu, cudaStream_t st) {
    MS_REQUIRE(dp_connected, "dp_update: peers not connected");
    size_t b = 0, e = n_params;
    if (group >= 0) { MS_REQUIRE(group < n_groups, "dp_update: bad group"); b = group_begin[group]; e = group_end[group]; }
    const size_t n = e - b;
    MS_REQUIRE((n & 3) == 0 && (b & 3) == 0 && n + 4 <= dp_cap_floats, "dp_update: range not 16-byte granular / too large");
    const unsigned blocks = (unsigned)std::max<size_t>(1, std::min<size_t>(cdivz(n / 4, 256), NUM_SMS * 2));
    dp_pack_kernel<<<blocks, 256, 0, st>>>(dp_state, dp_world, dp_rank, Gr + b, n, scalars, dp_xbuf);
    DpPeers peers;
    memset(&peers, 0, sizeof peers);
    for (int r = 0; r < dp_world; ++r) { peers.xbuf[r] = dp_peer_xbuf[r]; peers.state[r] = dp_peer_state[r]; }
    dp_reduce_update_kernel<<<blocks, 256, 0, st>>>(dp_state, peers, dp_world, dp_rank, (unsigned)(group + 2), n, Wt + b, Gr + b,
                                                    Mo + b, lr, mu, 1.f / (float)dp_world, scalars);
    if (check_launch("dp_update", 2)) return -1;
    return prep_layers(group, st);
}

int Engine::dp_error(unsigned int* out) {
    MS_REQUIRE(dp_state != nullptr, "dp_error: no exchange state");
    MS_CHECK_CUDA(cudaMemcpy(out, &dp_state->error, sizeof(unsigned int), cudaMemcpyDeviceToHost));
    return 0;
}

}  // namespace ms
