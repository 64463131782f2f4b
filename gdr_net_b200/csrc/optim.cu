// Fused Ranger step (SURVEY.md 8f row f-2): gradient centralisation + RAdam + Lookahead for ALL parameter tensors in ONE
// launch.  Replaces the reference's per-parameter Python loop, lib/torch_utils/solver/ranger.py:100-200 (~12 ATen
// kernels x 148 tensors per step), and the multi-tensor torch._foreach restatement of round 1.
//
// HBM-bound: per step the kernel reads g, p, m, v and writes p, m, v once (28 B / parameter; +8 B on the every-k-th
// lookahead step); the centralisation's second read of a gradient row hits L1/L2.  35.05 M parameters -> 0.98 GB -> ~0.3 ms
// at H100 HBM3 bandwidth.
//
// Work decomposition: a device-resident table of per-tensor jobs and a flat list of block descriptors built once by the
// host (gdr_net_b200/solver.py).  Tensors with dim > 1 are centralised per output row (mean over dims 1..): rows of up to
// 2048 elements are owned by one warp (8 rows in flight per block), longer rows by the whole block.
#include "gdrn_internal.h"
#include "ptx.cuh"

namespace gdrn {

struct RangerJob {     // 64 bytes
    float* p;          // parameter (fp32, updated in place)
    const float* g;    // gradient
    float* m;          // exp_avg
    float* v;          // exp_avg_sq
    float* slow;       // lookahead slow weights
    long numel;
    int row_len;       // > 0: gradient centralisation over rows of this length (numel % row_len == 0); 0: none
    int pad[3];
};
static_assert(sizeof(RangerJob) == 64, "RangerJob layout");

struct RangerBlock {  // 16 bytes
    int job;
    int count;   // rows (row_len > 0) or elements (row_len == 0) handled by this block
    long begin;  // first row / first element
};

struct RangerHyper {
    float beta1, beta2, eps, alpha, g_scale;
    float step_lr;  // step_size * lr of the param group (RAdam rectification folded in by the host)
    float wd_lr;    // weight_decay * lr
    int adaptive;   // N_sma > threshold: p -= step_lr * m / (sqrt(v) + eps); else p -= step_lr * m
    int lookahead;  // step % k == 0: slow += alpha * (p - slow); p = slow
};

__device__ __forceinline__ void ranger_update(const RangerJob& J, const RangerHyper& h, long i, float g) {
    const float m = h.beta1 * J.m[i] + (1.f - h.beta1) * g;
    const float v = h.beta2 * J.v[i] + (1.f - h.beta2) * g * g;
    J.m[i] = m;
    J.v[i] = v;
    float p = J.p[i];
    if (h.wd_lr != 0.f) p -= h.wd_lr * p;
    p -= h.adaptive ? h.step_lr * (m / (sqrtf(v) + h.eps)) : h.step_lr * m;
    if (h.lookahead) {
        const float s = J.slow[i] + h.alpha * (p - J.slow[i]);
        J.slow[i] = s;
        p = s;
    }
    J.p[i] = p;
}

__global__ void __launch_bounds__(256) ranger_step_kernel(const RangerJob* __restrict__ jobs, const RangerBlock* __restrict__ blocks,
                                                          const RangerHyper h) {
    const RangerBlock B = blocks[blockIdx.x];
    const RangerJob J = jobs[B.job];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (J.row_len == 0) {
        const long end = B.begin + B.count;
        for (long i = B.begin + threadIdx.x; i < end; i += 256) ranger_update(J, h, i, J.g[i] * h.g_scale);
        return;
    }
    const int L = J.row_len;
    const float invL = 1.f / (float)L;
    if (L <= 2048) {  // one warp per row
        for (int r = warp; r < B.count; r += 8) {
            const long base = (B.begin + r) * (long)L;
            float s = 0.f;
            for (int j = lane; j < L; j += 32) s += J.g[base + j];
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            const float mean = s * invL;
            for (int j = lane; j < L; j += 32) ranger_update(J, h, base + j, (J.g[base + j] - mean) * h.g_scale);
        }
    } else {  // the whole block per row
        __shared__ float red[8];
        for (int r = 0; r < B.count; ++r) {
            const long base = (B.begin + r) * (long)L;
            float s = 0.f;
            for (int j = threadIdx.x; j < L; j += 256) s += J.g[base + j];
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            __syncthreads();  // red[] of the previous row fully consumed
            if (lane == 0) red[warp] = s;
            __syncthreads();
            float tot = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) tot += red[w];
            const float mean = tot * invL;
            for (int j = threadIdx.x; j < L; j += 256) ranger_update(J, h, base + j, (J.g[base + j] - mean) * h.g_scale);
        }
    }
}

// x[i] *= s (removal of the static fp16 loss scale from a slice of the flat fp32 gradient buffer); `head` unaligned leading
// elements and the tail are handled by block 0, the 16-byte aligned body with float4 accesses
__global__ void scale_f32_kernel(float* __restrict__ x, long head, long n4, long n, float s) {
    pdl_ew_entry();
    float4* body = reinterpret_cast<float4*>(x + head);
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        float4 q = body[i];
        q.x *= s; q.y *= s; q.z *= s; q.w *= s;
        body[i] = q;
    }
    if (blockIdx.x == 0) {
        if (threadIdx.x < head) x[threadIdx.x] *= s;
        for (long i = head + n4 * 4 + threadIdx.x; i < n; i += blockDim.x) x[i] *= s;
    }
}

}  // namespace gdrn

using namespace gdrn;

extern "C" int gdrn_ranger_step(const void* jobs_dev, const void* blocks_dev, int nblocks, float step_lr, float wd_lr, float beta1,
                                float beta2, float eps, float alpha, float grad_scale, int adaptive, int lookahead,
                                void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (nblocks <= 0) return set_error(GDRN_ERR_ARG, "ranger_step: empty block list");
    RangerHyper h;
    h.beta1 = beta1;
    h.beta2 = beta2;
    h.eps = eps;
    h.alpha = alpha;
    h.g_scale = grad_scale;
    h.step_lr = step_lr;
    h.wd_lr = wd_lr;
    h.adaptive = adaptive;
    h.lookahead = lookahead;
    ranger_step_kernel<<<nblocks, 256, 0, stream>>>(reinterpret_cast<const RangerJob*>(jobs_dev),
                                                    reinterpret_cast<const RangerBlock*>(blocks_dev), h);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_scale_f32(float* x, long n, float s, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if ((reinterpret_cast<uintptr_t>(x) & 3) != 0) return set_error(GDRN_ERR_ARG, "scale_f32: pointer must be 4-byte aligned");
    long head = (long)((16 - (reinterpret_cast<uintptr_t>(x) & 15)) & 15) / 4;
    if (head > n) head = n;
    const long n4 = (n - head) / 4;
    long g = (n4 + 255) / 256;
    const long cap = (long)num_sms() * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    GDRN_LAUNCH_PDL(scale_f32_kernel, (int)g, 256, 0, stream, x, head, n4, n, s);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
