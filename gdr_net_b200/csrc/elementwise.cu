// HBM-bound elementwise / normalisation kernels of the GDR-Net hot path (NHWC, bf16 hi[/lo] planes,
// fp32 math, 16-byte vector accesses: one thread = 8 consecutive channels).
//
// Reference ops replaced (all ATen / cuDNN library kernels today, SURVEY.md 2.2 K2, K9, K20):
//   nn.BatchNorm2d train/eval + ReLU (+ residual add)        resnet_backbone.py:69-76, torchvision BasicBlock
//   nn.MaxPool2d(3, 2, 1)                                    resnet_backbone.py:72
//   nn.UpsamplingBilinear2d(scale_factor=2) (align_corners)  cdpn_rot_head_region.py:102
//   nn.GroupNorm(32, 128) + ReLU                             conv_pnp_net.py:76-80
// and their autograd backward.
#include <stdlib.h>

#include "gdrn_internal.h"
#include "ptx.cuh"

namespace gdrn {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void unpack8(const uint4& q, float (&f)[8]) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        unpack_hi2(w[j], f[2 * j], f[2 * j + 1]);
    }
}
// value = hi (+ lo)
__device__ __forceinline__ void load8(const bf16* hi, const bf16* lo, long off8, float (&f)[8]) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(hi) + off8), f);
    if (lo != nullptr) {
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(lo) + off8);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float a, b;
            unpack_lo2(w[j], a, b);
            f[2 * j] += a;
            f[2 * j + 1] += b;
        }
    }
}
__device__ __forceinline__ void store8(bf16* hi, bf16* lo, long off8, const float (&f)[8]) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        split2(f[2 * j], f[2 * j + 1], h[j], l[j]);
    }
    reinterpret_cast<uint4*>(hi)[off8] = make_uint4(h[0], h[1], h[2], h[3]);
    if (lo != nullptr) reinterpret_cast<uint4*>(lo)[off8] = make_uint4(l[0], l[1], l[2], l[3]);
}

static inline int ew_grid(long total, int block) {
    long g = (total + block - 1) / block;
    const long cap = (long)num_sms() * 8;
    return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}
// for kernels with a per-thread prologue (per-channel coefficients): at least `per_thread` items per thread so the
// prologue is amortised on small tensors (a 4 MB layer4 tensor must not pay 300K threads x 16 coefficient loads)
static inline int ew_grid_amortised(long total, int block, int per_thread) {
    long g = (total + (long)block * per_thread - 1) / ((long)block * per_thread);
    const long cap = (long)num_sms() * 8;
    return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

// ------------------------------------------------------------------------------------------------
// BatchNorm statistics -> per-channel scale/shift (+ running-stat update)
// ------------------------------------------------------------------------------------------------
__global__ void bn_finalize_kernel(const float* __restrict__ stats, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* running_mean, float* running_var,
                                   float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ mean_out,
                                   float* __restrict__ invstd_out, int C, float count, float eps, float momentum, int train) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float mean, var;
    if (train) {
        const double m = (double)stats[c] / count;
        double v = (double)stats[C + c] / count - m * m;
        if (v < 0) v = 0;
        mean = (float)m;
        var = (float)v;
        if (running_mean != nullptr) {
            running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
            const float unbiased = count > 1.f ? var * (count / (count - 1.f)) : var;
            running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
        }
    } else {
        mean = running_mean[c];
        var = running_var[c];
    }
    const float invstd = rsqrtf(var + eps);
    const float sc = gamma[c] * invstd;
    scale[c] = sc;
    shift[c] = beta[c] - mean * sc;
    if (mean_out != nullptr) {
        mean_out[c] = mean;
        invstd_out[c] = invstd;
    }
}

// Eval-mode BatchNorm folding for ALL layers in one launch: scale = gamma / sqrt(running_var + eps), shift = beta -
// running_mean * scale.  The scales are multiplied into the packed conv weights (pack.cu row_scale), the shifts become
// the conv epilogue's bias: inference runs conv + BN + (residual) + ReLU as ONE kernel per layer (north_star "fused
// conv+BN+ReLU epilogues"; reference inference caller gdrn_evaluator.py:568-580).
struct BnFoldJob {  // 64 bytes
    const float* gamma;
    const float* beta;
    const float* mean;
    const float* var;
    float* scale;
    float* shift;
    int C;
    float eps;
    long pad;
};
__global__ void bn_fold_batched_kernel(const BnFoldJob* __restrict__ jobs) {
    const BnFoldJob J = jobs[blockIdx.x];
    for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < J.C; c += gridDim.y * blockDim.x) {
        const float sc = J.gamma[c] * rsqrtf(J.var[c] + J.eps);
        J.scale[c] = sc;
        J.shift[c] = J.beta[c] - J.mean[c] * sc;
    }
}

// ------------------------------------------------------------------------------------------------
// BatchNorm forward.  Design notes: keeping unpacked fp32 arrays live across the loads costs registers and with them the
// warps that keep HBM busy (115 registers -> 2 blocks/SM).  The 16-byte loads
// stay PACKED in registers while in flight (4 per tensor), per-channel coefficients live in shared memory, and the
// kernels are templated on "has lo plane" / "has residual" so unused operands cost nothing.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld16(const bf16* p, long off8) { return __ldg(reinterpret_cast<const uint4*>(p) + off8); }
__device__ __forceinline__ void unpack8_lo(const uint4& q, float (&f)[8]) {  // adds the lo plane
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float a, b;
        unpack_lo2(w[j], a, b);
        f[2 * j] += a;
        f[2 * j + 1] += b;
    }
}

// y = [relu](x * sc[c] + sh[c] [+ res]);  s_sc / s_sh: shared memory [C]
// mask_out (optional, with relu): one byte per 8-channel group, bit j = [pre-activation of channel j > 0].  BatchNorm
// backward reads this byte instead of the 16-byte activation group to rebuild the ReLU mask (3.75 of its 14 B / element).
template <bool LO, bool RES>
__device__ __forceinline__ void bn_apply_loop(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo,
                                              const bf16* __restrict__ r_hi, const bf16* __restrict__ r_lo,
                                              bf16* __restrict__ y_hi, bf16* __restrict__ y_lo, const float* s_sc,
                                              const float* s_sh, long total, int cg, int relu, uint8_t* __restrict__ mask_out,
                                              bool rev = false) {
    // rev: walk the tensor from its END to its start.  The producing GEMM wrote it front to back, so for tensors larger than
    // the 50 MB L2 the freshest ~40 MB are the tail; this kernel's own output then leaves its HEAD in L2, which is where the
    // consuming GEMM starts (total is a multiple of cg, so a thread's channel group stays fixed in both directions).
    const long stride = (long)gridDim.x * blockDim.x;
    const long first = blockIdx.x * (long)blockDim.x + threadIdx.x;
    const int c0 = (rev ? cg - 1 - (int)(first % cg) : (int)(first % cg)) * 8;
    for (long idx = first; idx < total; idx += 4 * stride) {
        uint4 xr[4], xl[4], rr[4], rl[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const long it0 = idx + t * stride;
            const long it = rev ? total - 1 - it0 : it0;
            if (it0 < total) {
                xr[t] = ld16(x_hi, it);
                if (LO) xl[t] = ld16(x_lo, it);
                if (RES) {
                    rr[t] = ld16(r_hi, it);
                    if (LO) rl[t] = ld16(r_lo, it);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const long it0 = idx + t * stride;
            const long it = rev ? total - 1 - it0 : it0;
            if (it0 < total) {
                float v[8];
                unpack8(xr[t], v);
                if (LO) unpack8_lo(xl[t], v);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], s_sc[c0 + j], s_sh[c0 + j]);
                if (RES) {
                    float r[8];
                    unpack8(rr[t], r);
                    if (LO) unpack8_lo(rl[t], r);
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] += r[j];
                }
                if (relu) {
                    if (mask_out != nullptr) {
                        uint32_t bits = 0;
#pragma unroll
                        for (int j = 0; j < 8; ++j) bits |= (v[j] > 0.f ? 1u : 0u) << j;
                        mask_out[it] = (uint8_t)bits;
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
                }
                store8(y_hi, LO ? y_lo : nullptr, it, v);
            }
        }
    }
}

template <bool LO, bool RES>
__global__ void __launch_bounds__(256, 4) bn_act_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo,
                                                        const bf16* __restrict__ r_hi, const bf16* __restrict__ r_lo,
                                                        bf16* __restrict__ y_hi, bf16* __restrict__ y_lo,
                                                        const float* __restrict__ scale, const float* __restrict__ shift,
                                                        long rows, int C, int relu) {
    pdl_ew_entry();
    __shared__ float s_sc[512], s_sh[512];
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        s_sc[c] = scale[c];
        s_sh[c] = shift[c];
    }
    __syncthreads();
    bn_apply_loop<LO, RES>(x_hi, x_lo, r_hi, r_lo, y_hi, y_lo, s_sc, s_sh, rows * (C / 8), C / 8, relu, nullptr);
}

// finalize + apply in one kernel: scale/shift from the conv epilogue's (sum, sum^2) (train) or the running statistics
// (eval); block 0 stores mean/invstd for backward and updates the running statistics like nn.BatchNorm2d.
template <bool LO, bool RES>
__global__ void __launch_bounds__(256, 4) bn_fwd_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo,
                                                        const bf16* __restrict__ r_hi, const bf16* __restrict__ r_lo,
                                                        bf16* __restrict__ y_hi, bf16* __restrict__ y_lo,
                                                        const float* __restrict__ stats, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float* running_mean, float* running_var,
                                                        float* __restrict__ mean_out, float* __restrict__ invstd_out, long rows,
                                                        int C, float eps, float momentum, int train, int relu,
                                                        uint8_t* __restrict__ mask_out, int rev) {
    pdl_ew_entry();
    __shared__ float s_sc[512], s_sh[512];
    const float count = (float)rows;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float mean, var;
        if (train) {
            // train & 2: the statistics were accumulated in double (GEMM epilogue with kActStatsF64)
            const double* s64 = reinterpret_cast<const double*>(stats);
            const double m = ((train & 2) ? s64[c] : (double)stats[c]) / count;
            double v = ((train & 2) ? s64[C + c] : (double)stats[C + c]) / count - m * m;
            if (v < 0) v = 0;
            mean = (float)m;
            var = (float)v;
        } else {
            mean = running_mean[c];
            var = running_var[c];
        }
        const float invstd = rsqrtf(var + eps);
        const float sc = gamma[c] * invstd;
        s_sc[c] = sc;
        s_sh[c] = beta[c] - mean * sc;
        if (blockIdx.x == 0) {
            if (mean_out != nullptr) {
                mean_out[c] = mean;
                invstd_out[c] = invstd;
            }
            if (train && running_mean != nullptr) {
                running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
                const float unbiased = count > 1.f ? var * (count / (count - 1.f)) : var;
                running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
            }
        }
    }
    __syncthreads();
    bn_apply_loop<LO, RES>(x_hi, x_lo, r_hi, r_lo, y_hi, y_lo, s_sc, s_sh, rows * (C / 8), C / 8, relu, mask_out, rev != 0);
}


// (channel group, x, y, image) of a flat NHWC index with 32-bit arithmetic (every tensor of the step has < 2^31 groups;
// 64-bit div / mod costs ~100 instructions each and dominated the gather kernels)
struct Pix {
    int g, x, y, b;
};
// every tensor of this network has power-of-two channel groups / widths / heights: shifts and masks instead of three
// 32-bit divisions (the gather kernels are instruction-bound, not bandwidth-bound)
__device__ __forceinline__ bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }
__device__ __forceinline__ Pix decode_pix(long idx, int cg, int W, int H) {
    unsigned t = (unsigned)idx;
    Pix p;
    if (is_pow2(cg) && is_pow2(W) && is_pow2(H)) {  // block-uniform branch
        const int lc = 31 - __clz(cg), lw = 31 - __clz(W), lh = 31 - __clz(H);
        p.g = (int)(t & (unsigned)(cg - 1));
        t >>= lc;
        p.x = (int)(t & (unsigned)(W - 1));
        t >>= lw;
        p.y = (int)(t & (unsigned)(H - 1));
        p.b = (int)(t >> lh);
        return p;
    }
    unsigned q = t / (unsigned)cg;
    p.g = (int)(t - q * (unsigned)cg);
    t = q;
    q = t / (unsigned)W;
    p.x = (int)(t - q * (unsigned)W);
    t = q;
    q = t / (unsigned)H;
    p.y = (int)(t - q * (unsigned)H);
    p.b = (int)q;
    return p;
}

// ------------------------------------------------------------------------------------------------
// MaxPool 3x3 s2 p1 (first maximum in row-major window order wins, like ATen)
// ------------------------------------------------------------------------------------------------
__global__ void maxpool_fwd_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo, bf16* __restrict__ y_hi,
                                   bf16* __restrict__ y_lo, uint8_t* __restrict__ arg_out, int B, int H, int W, int C) {
    pdl_ew_entry();
    const int cg = C / 8, Ho = H / 2, Wo = W / 2;
    const long total = (long)B * Ho * Wo * cg;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const Pix px = decode_pix(idx, cg, Wo, Ho);
        const int g = px.g, ox = px.x, oy = px.y, b = px.b;
        float m[8];
        uint32_t arg[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            m[j] = -INFINITY;
            arg[j] = 0;
        }
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const int iy = oy * 2 + dy - 1;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int ix = ox * 2 + dx - 1;
                if (ix < 0 || ix >= W) continue;
                float v[8];
                load8(x_hi, x_lo, (((long)b * H + iy) * W + ix) * cg + g, v);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (v[j] > m[j]) {
                        m[j] = v[j];
                        arg[j] = dy * 3 + dx;
                    }
            }
        }
        store8(y_hi, y_lo, idx, m);
        if (arg_out != nullptr) {
            uint2 packed;
            packed.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
            packed.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | (arg[7] << 24);
            reinterpret_cast<uint2*>(arg_out)[idx] = packed;
        }
    }
}

// dx[iy,ix] = sum of g over the (<=4) windows whose saved arg-max (window-local code dy*3+dx, first maximum) is (iy,ix)
__global__ void maxpool_bwd_kernel(const uint8_t* __restrict__ arg_in, const bf16* __restrict__ g_hi,
                                   const bf16* __restrict__ g_lo, bf16* __restrict__ dx_hi, bf16* __restrict__ dx_lo, int B, int H,
                                   int W, int C) {
    pdl_ew_entry();
    const int cg = C / 8, Ho = H / 2, Wo = W / 2;
    const long total = (long)B * H * W * cg;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const Pix px = decode_pix(idx, cg, W, H);
        const int g = px.g, ix = px.x, iy = px.y, b = px.b;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        // windows (oy, ox) with oy*2-1 <= iy <= oy*2+1: oy in {iy/2, (iy+1)/2} (one window per axis for even iy, two for odd).
        // All four candidates' loads are issued before any is consumed (the loop form serialised 8 dependent L2 round trips).
        const int oyA = iy >> 1, oyB = (iy + 1) >> 1, oxA = ix >> 1, oxB = (ix + 1) >> 1;
        const bool vyB = (oyB != oyA) && (oyB < Ho), vxB = (oxB != oxA) && (oxB < Wo);
        const int oys[2] = {oyA, vyB ? oyB : oyA}, oxs[2] = {oxA, vxB ? oxB : oxA};
        uint2 codes[4];
        uint4 gh[4], gl[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const long o = (((long)b * Ho + oys[q >> 1]) * Wo + oxs[q & 1]) * cg + g;
            codes[q] = __ldg(reinterpret_cast<const uint2*>(arg_in) + o);
            gh[q] = ld16(g_hi, o);
            if (g_lo != nullptr) gl[q] = ld16(g_lo, o);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const bool valid = ((q >> 1) == 0 || vyB) && ((q & 1) == 0 || vxB);
            if (!valid) continue;
            const uint32_t code = (uint32_t)((iy - (oys[q >> 1] * 2 - 1)) * 3 + (ix - (oxs[q & 1] * 2 - 1)));
            float gv[8];
            unpack8(gh[q], gv);
            if (g_lo != nullptr) unpack8_lo(gl[q], gv);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t aj = ((j < 4 ? codes[q].x : codes[q].y) >> (8 * (j & 3))) & 0xffu;
                if (aj == code) acc[j] += gv[j];
            }
        }
        store8(dx_hi, dx_lo, idx, acc);
    }
}

// ------------------------------------------------------------------------------------------------
// Bilinear x2 upsampling, align_corners=True
// ------------------------------------------------------------------------------------------------
__global__ void upsample2x_fwd_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo, bf16* __restrict__ y_hi,
                                      bf16* __restrict__ y_lo, int B, int H, int W, int C) {
    pdl_ew_entry();
    const int cg = C / 8, Ho = 2 * H, Wo = 2 * W;
    const float sh = (float)(H - 1) / (float)(Ho - 1), sw = (float)(W - 1) / (float)(Wo - 1);
    const long total = (long)B * Ho * Wo * cg;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const Pix px = decode_pix(idx, cg, Wo, Ho);
        const int g = px.g, ox = px.x, oy = px.y, b = px.b;
        const float fy = sh * oy, fx = sw * ox;
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
        const float ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
        float v00[8], v01[8], v10[8], v11[8], o[8];
        const long base = (long)b * H;
        load8(x_hi, x_lo, ((base + y0) * W + x0) * cg + g, v00);
        load8(x_hi, x_lo, ((base + y0) * W + x1) * cg + g, v01);
        load8(x_hi, x_lo, ((base + y1) * W + x0) * cg + g, v10);
        load8(x_hi, x_lo, ((base + y1) * W + x1) * cg + g, v11);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = ly0 * (lx0 * v00[j] + lx1 * v01[j]) + ly1 * (lx0 * v10[j] + lx1 * v11[j]);
        store8(y_hi, y_lo, idx, o);
    }
}

// gather form of the transpose: dx[iy,ix] = sum_{oy,ox} w(oy->iy) * w(ox->ix) * g[oy,ox]
__global__ void upsample2x_bwd_kernel(const bf16* __restrict__ g_hi, const bf16* __restrict__ g_lo, bf16* __restrict__ dx_hi,
                                      bf16* __restrict__ dx_lo, int B, int H, int W, int C) {
    pdl_ew_entry();
    const int cg = C / 8, Ho = 2 * H, Wo = 2 * W;
    const float sh = (float)(H - 1) / (float)(Ho - 1), sw = (float)(W - 1) / (float)(Wo - 1);
    const long total = (long)B * H * W * cg;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const Pix px = decode_pix(idx, cg, W, H);
        const int g = px.g, ix = px.x, iy = px.y, b = px.b;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        // output rows whose source coordinate sh*oy lies in [iy-1, iy+1): oy in [2iy-2, 2iy+3] since 1/sh is in (2, 2.07];
        // the exact weight computed below is zero for the one or two extra candidates.  Column weights do not depend on
        // the row, so they are computed once; the (<= 6) loads of a row are issued together.
        const int oy0 = 2 * iy - 2, ox0 = 2 * ix - 2;
        float wxs[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) {
            const int ox = ox0 + c;
            float wx = 0.f;
            if (ox >= 0 && ox < Wo) {
                const float fx = sw * ox;
                const int x0 = (int)fx;
                const int x1 = x0 + (x0 < W - 1 ? 1 : 0);
                const float lx1 = fx - x0, lx0 = 1.f - lx1;
                if (x0 == ix) wx += lx0;
                if (x1 == ix) wx += lx1;
            }
            wxs[c] = wx;
        }
        for (int r = 0; r < 6; ++r) {
            const int oy = oy0 + r;
            if (oy < 0 || oy >= Ho) continue;
            const float fy = sh * oy;
            const int y0 = (int)fy;
            const int y1 = y0 + (y0 < H - 1 ? 1 : 0);
            const float ly1 = fy - y0, ly0 = 1.f - ly1;
            float wy = 0.f;
            if (y0 == iy) wy += ly0;
            if (y1 == iy) wy += ly1;
            if (wy == 0.f) continue;
            const long rowbase = (((long)b * Ho + oy) * Wo + ox0) * cg + g;
            uint4 vh[6], vl[6];
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                if (wxs[c] != 0.f) {
                    vh[c] = ld16(g_hi, rowbase + (long)c * cg);
                    if (g_lo != nullptr) vl[c] = ld16(g_lo, rowbase + (long)c * cg);
                }
            }
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                if (wxs[c] != 0.f) {
                    float gv[8];
                    unpack8(vh[c], gv);
                    if (g_lo != nullptr) unpack8_lo(vl[c], gv);
                    const float w = wy * wxs[c];
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = fmaf(w, gv[j], acc[j]);
                }
            }
        }
        store8(dx_hi, dx_lo, idx, acc);
    }
}

// ------------------------------------------------------------------------------------------------
// zero insertion (stride-2 transposed convs as stride-1 convs) and its transpose
//   mode 0: y[2i,2j] = x[i,j], 0 elsewhere (y is [B,2H,2W,C]);  mode 1: y[i,j] = x[2i,2j] (x is [B,2H,2W,C])
// ------------------------------------------------------------------------------------------------
__global__ void zero_insert_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo, bf16* __restrict__ y_hi,
                                   bf16* __restrict__ y_lo, int B, int H, int W, int C, int mode) {
    pdl_ew_entry();
    const int cg = C / 8;
    const int Hy = mode == 0 ? 2 * H : H, Wy = mode == 0 ? 2 * W : W;
    const long total = (long)B * Hy * Wy * cg;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const int g = (int)(idx % cg);
        long t = idx / cg;
        const int x = (int)(t % Wy);
        t /= Wy;
        const int y = (int)(t % Hy);
        const int b = (int)(t / Hy);
        uint4 h = make_uint4(0, 0, 0, 0), l = make_uint4(0, 0, 0, 0);
        if (mode == 0) {
            if (((x | y) & 1) == 0) {
                const long s = (((long)b * H + (y >> 1)) * W + (x >> 1)) * cg + g;
                h = __ldg(reinterpret_cast<const uint4*>(x_hi) + s);
                if (x_lo != nullptr) l = __ldg(reinterpret_cast<const uint4*>(x_lo) + s);
            }
        } else {
            const long s = (((long)b * 2 * H + 2 * y) * 2 * W + 2 * x) * cg + g;
            h = __ldg(reinterpret_cast<const uint4*>(x_hi) + s);
            if (x_lo != nullptr) l = __ldg(reinterpret_cast<const uint4*>(x_lo) + s);
        }
        reinterpret_cast<uint4*>(y_hi)[idx] = h;
        if (y_lo != nullptr) reinterpret_cast<uint4*>(y_lo)[idx] = l;
    }
}

// ------------------------------------------------------------------------------------------------
// BatchNorm(+ReLU) backward.  g = (ga [+ gb]) * [y > 0];  xhat = (u - mean) * invstd
//   reduce: sums[0][c] = sum g, sums[1][c] = sum g * xhat
//   apply : du = gamma*invstd * (g - sums0/n - xhat * sums1/n);  optional g_out = g;  dgamma = sums1, dbeta = sums0
// ------------------------------------------------------------------------------------------------
constexpr int kBnBwdThreads = 256;
constexpr int kRedRows = 4;  // rows in flight per thread of the reduction pass: more loads in flight per thread for the HBM-bound reads

// masked gradient of one 8-channel group: g = (ga [+ gb]) * [y > 0]
template <bool LO>
__device__ __forceinline__ void masked_grad(const uint4& gah, const uint4& gal, const uint4& gbh, const uint4& gbl, const uint4& yh,
                                            bool has_gb, bool has_y, float (&g)[8], bool has_bits = false, uint32_t bits = 0) {
    unpack8(gah, g);
    if (LO) unpack8_lo(gal, g);
    if (has_gb) {
        float t[8];
        unpack8(gbh, t);
        if (LO) unpack8_lo(gbl, t);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] += t[j];
    }
    if (has_bits) {
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = ((bits >> j) & 1u) ? g[j] : 0.f;
    } else if (has_y) {
        float y[8];
        unpack8(yh, y);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = y[j] > 0.f ? g[j] : 0.f;
    }
}
// 8 consecutive per-channel constants from shared memory with two 16-byte loads (the arrays are 16-byte aligned, c0 % 8 == 0)
__device__ __forceinline__ void lds8(const float* p, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// ReLU mask recomputed from the BN input: [sc*u + sh > 0] with the forward's own scale / shift (bn_fwd_kernel), so the
// activation y need not be read back (plain conv-BN-ReLU layers: 2 of the 14 bytes per element of BN backward)
__device__ __forceinline__ void mask_from_u(const float (&u)[8], const float* sc_, const float* sh_, float (&g)[8]) {
    float sc[8], sh[8];
    lds8(sc_, sc);
    lds8(sh_, sh);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = fmaf(sc[j], u[j], sh[j]) > 0.f ? g[j] : 0.f;
}

template <bool LO, bool MASKU>
__global__ void __launch_bounds__(kBnBwdThreads, 2) bn_bwd_reduce_kernel(
    const bf16* __restrict__ ga_hi, const bf16* __restrict__ ga_lo, const bf16* __restrict__ gb_hi,
    const bf16* __restrict__ gb_lo, const bf16* __restrict__ y_hi, const bf16* __restrict__ u_hi,
    const bf16* __restrict__ u_lo, const float* __restrict__ mean, const float* __restrict__ invstd,
    const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ sums, long rows, int C,
    const uint8_t* __restrict__ mask_in, float* __restrict__ partial_out) {
    pdl_ew_entry();
    // block = (C/8) channel groups x rpb row lanes
    const int cg = C / 8;
    const int rpb = kBnBwdThreads / cg;  // cg in {8,16,32,64}: always divides 256
    const int g = threadIdx.x % cg;
    const int rl = threadIdx.x / cg;
    __shared__ __align__(16) float s_mu[512], s_is[512], s_sc[512], s_sh[512];
    __shared__ float red[2][kBnBwdThreads][8 + 1];
    for (int c = threadIdx.x; c < C; c += kBnBwdThreads) {
        s_mu[c] = mean[c];
        s_is[c] = invstd[c];
        if (MASKU) {
            const float sc = gamma[c] * invstd[c];
            s_sc[c] = sc;
            s_sh[c] = beta[c] - mean[c] * sc;
        }
    }
    __syncthreads();
    const bool has_bits = !MASKU && mask_in != nullptr;
    const bool has_gb = gb_hi != nullptr, has_y = !MASKU && !has_bits && y_hi != nullptr;
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    const long rstride = (long)gridDim.x * rpb;
    for (long r0 = (long)blockIdx.x * rpb + rl; r0 < rows; r0 += kRedRows * rstride) {
        uint4 gah[kRedRows], gal[kRedRows], gbh[kRedRows], gbl[kRedRows], yh[kRedRows], uh[kRedRows], ul[kRedRows];
        uint32_t mb[kRedRows] = {};
#pragma unroll
        for (int t = 0; t < kRedRows; ++t) {
            const long r = r0 + t * rstride;
            if (r < rows) {
                const long off = r * cg + g;
                gah[t] = ld16(ga_hi, off);
                uh[t] = ld16(u_hi, off);
                if (has_bits) mb[t] = __ldg(mask_in + off);
                if (has_y) yh[t] = ld16(y_hi, off);
                if (has_gb) gbh[t] = ld16(gb_hi, off);
                if (LO) {
                    gal[t] = ld16(ga_lo, off);
                    ul[t] = ld16(u_lo, off);
                    if (has_gb) gbl[t] = ld16(gb_lo, off);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < kRedRows; ++t) {
            const long r = r0 + t * rstride;
            if (r < rows) {
                float gv[8], u[8];
                masked_grad<LO>(gah[t], gal[t], gbh[t], gbl[t], yh[t], has_gb, has_y, gv, has_bits, mb[t]);
                unpack8(uh[t], u);
                if (LO) unpack8_lo(ul[t], u);
                if (MASKU) mask_from_u(u, s_sc + g * 8, s_sh + g * 8, gv);
                float mu[8], is[8];
                lds8(s_mu + g * 8, mu);
                lds8(s_is + g * 8, is);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    s0[j] += gv[j];
                    s1[j] = fmaf(gv[j], (u[j] - mu[j]) * is[j], s1[j]);
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[0][threadIdx.x][j] = s0[j];
        red[1][threadIdx.x][j] = s1[j];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 2 * C; t += kBnBwdThreads) {
        const int which = t / C, c = t % C;
        const int gg = c / 8, j = c % 8;
        float a = 0.f;
        for (int q = 0; q < rpb; ++q) a += red[which][q * cg + gg][j];
        // deterministic mode: per-block partials, summed in block order by sum_partials_kernel (no atomics anywhere)
        if (partial_out != nullptr) partial_out[((long)blockIdx.x * 2 + which) * C + c] = a;
        else atomicAdd(sums + which * C + c, a);
    }
}

// ------------------------------------------------------------------------------------------------
// Deterministic reductions (Engine.deterministic / GDRN_DETERMINISTIC=1): two-stage, fixed work decomposition, fixed
// summation order, no atomics -- bit-identical results run to run (the default path accumulates the BatchNorm batch
// statistics with fp32 atomics from the GEMM epilogues and the backward sums with atomics across blocks).
// ------------------------------------------------------------------------------------------------
// stage 1 of the BatchNorm batch statistics: partials[blk][0][c] = sum x, [blk][1][c] = sum x^2 over the block's rows
template <bool LO>
__global__ void __launch_bounds__(kBnBwdThreads, 3) bn_stats_partial_kernel(const bf16* __restrict__ u_hi, const bf16* __restrict__ u_lo,
                                                                            float* __restrict__ partials, long rows, int C) {
    const int cg = C / 8;
    const int rpb = kBnBwdThreads / cg;
    const int g = threadIdx.x % cg, rl = threadIdx.x / cg;
    __shared__ float red[2][kBnBwdThreads][8 + 1];
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    const long rstride = (long)gridDim.x * rpb;
    for (long r = (long)blockIdx.x * rpb + rl; r < rows; r += rstride) {
        float v[8];
        const long off = r * cg + g;
        unpack8(ld16(u_hi, off), v);
        if (LO) unpack8_lo(ld16(u_lo, off), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s0[j] += v[j];
            s1[j] = fmaf(v[j], v[j], s1[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[0][threadIdx.x][j] = s0[j];
        red[1][threadIdx.x][j] = s1[j];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 2 * C; t += kBnBwdThreads) {
        const int which = t / C, c = t % C;
        float a = 0.f;
        for (int q = 0; q < rpb; ++q) a += red[which][q * cg + c / 8][c % 8];
        partials[((long)blockIdx.x * 2 + which) * C + c] = a;
    }
}
// stage 2: out[i] = sum over parts (in order) of partials[part][i]
__global__ void sum_partials_kernel(const float* __restrict__ partials, int nparts, int n, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double a = 0.0;
    for (int p = 0; p < nparts; ++p) a += (double)partials[(long)p * n + i];
    out[i] = (float)a;
}

// du = gamma*invstd*(g - mean(g) - xhat*mean(g*xhat)) = k1*g + k2*u + k3 with per-channel constants (shared memory)
template <bool LO, bool MASKU>
__global__ void __launch_bounds__(256, 4) bn_bwd_apply_kernel(
    const bf16* __restrict__ ga_hi, const bf16* __restrict__ ga_lo, const bf16* __restrict__ gb_hi,
    const bf16* __restrict__ gb_lo, const bf16* __restrict__ y_hi, const bf16* __restrict__ u_hi,
    const bf16* __restrict__ u_lo, const float* __restrict__ mean, const float* __restrict__ invstd,
    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ sums, bf16* __restrict__ du_hi,
    bf16* __restrict__ du_lo, bf16* __restrict__ gout_hi, bf16* __restrict__ gout_lo, float* __restrict__ dgamma,
    float* __restrict__ dbeta, long rows, int C, int train, const uint8_t* __restrict__ mask_in, int rev) {
    pdl_ew_entry();
    __shared__ __align__(16) float s_k1[512], s_k2[512], s_k3[512], s_sc[512], s_sh[512];
    const int cg = C / 8;
    const long total = rows * cg;
    const float inv_n = 1.f / (float)rows;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float is = invstd[c];
        const float k1 = gamma[c] * is;
        float k2 = 0.f, k3 = 0.f;
        if (train) {
            const float m0 = sums[c] * inv_n, m1 = sums[C + c] * inv_n;
            k2 = -k1 * is * m1;
            k3 = k1 * (mean[c] * is * m1 - m0);
        }
        s_k1[c] = k1;
        s_k2[c] = k2;
        s_k3[c] = k3;
        if (MASKU) {
            s_sc[c] = k1;  // gamma * invstd: the forward's scale
            s_sh[c] = beta[c] - mean[c] * k1;
        }
        if (blockIdx.x == 0 && dgamma != nullptr) {
            dbeta[c] = sums[c];
            dgamma[c] = sums[C + c];
        }
    }
    __syncthreads();
    const bool has_bits = !MASKU && mask_in != nullptr;
    const bool has_gb = gb_hi != nullptr, has_y = !MASKU && !has_bits && y_hi != nullptr, has_gout = gout_hi != nullptr;
    // rev: back to front (see bn_apply_loop): the reduction pass that ran just before left the TAIL of g / u in L2
    const long stride = (long)gridDim.x * blockDim.x;
    const long first = blockIdx.x * (long)blockDim.x + threadIdx.x;
    const int c0 = (rev ? cg - 1 - (int)(first % cg) : (int)(first % cg)) * 8;
    for (long idx = first; idx < total; idx += 2 * stride) {
        uint4 gah[2], gal[2], gbh[2], gbl[2], yh[2], uh[2], ul[2];
        uint32_t mb[2] = {0, 0};
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const long it0 = idx + t * stride;
            const long it = rev ? total - 1 - it0 : it0;
            if (it0 < total) {
                gah[t] = ld16(ga_hi, it);
                uh[t] = ld16(u_hi, it);
                if (has_bits) mb[t] = __ldg(mask_in + it);
                if (has_y) yh[t] = ld16(y_hi, it);
                if (has_gb) gbh[t] = ld16(gb_hi, it);
                if (LO) {
                    gal[t] = ld16(ga_lo, it);
                    ul[t] = ld16(u_lo, it);
                    if (has_gb) gbl[t] = ld16(gb_lo, it);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const long it0 = idx + t * stride;
            const long it = rev ? total - 1 - it0 : it0;
            if (it0 < total) {
                float gv[8], u[8], o[8];
                masked_grad<LO>(gah[t], gal[t], gbh[t], gbl[t], yh[t], has_gb, has_y, gv, has_bits, mb[t]);
                unpack8(uh[t], u);
                if (LO) unpack8_lo(ul[t], u);
                if (MASKU) mask_from_u(u, s_sc + c0, s_sh + c0, gv);
                float k1[8], k2[8], k3[8];
                lds8(s_k1 + c0, k1);
                lds8(s_k2 + c0, k2);
                lds8(s_k3 + c0, k3);
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = fmaf(k1[j], gv[j], fmaf(k2[j], u[j], k3[j]));
                store8(du_hi, LO ? du_lo : nullptr, it, o);
                if (has_gout) store8(gout_hi, LO ? gout_lo : nullptr, it, gv);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// GroupNorm(32 groups) + ReLU, one CTA per sample, tensor [HW][C] (C = 128 => 4 channels per group)
// ------------------------------------------------------------------------------------------------
// stats layout: [B][G][2] (mean, rstd).  Each thread owns one 8-channel column group (= 2 GN groups when C/G = 4)
// A sample is split over a CLUSTER of kGnCluster CTAs (one CTA per sample would use 64 of the 132 SMs at B = 64): each CTA owns a
// contiguous quarter of the rows, the per-group partial sums are exchanged through distributed shared memory.
constexpr int kGnCluster = 4;
__device__ __forceinline__ unsigned gn_cluster_rank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void gn_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ double gn_remote_f64(const double* local_smem_ptr, unsigned rank) {  // the same smem offset in CTA `rank`
    const unsigned a = (unsigned)__cvta_generic_to_shared(local_smem_ptr);
    unsigned ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a), "r"(rank));
    double v;
    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(ra) : "memory");
    return v;
}

__global__ void __launch_bounds__(256) gn_relu_fwd_kernel(const bf16* __restrict__ u_hi, const bf16* __restrict__ u_lo,
                                                          bf16* __restrict__ y_hi, bf16* __restrict__ y_lo,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          float* __restrict__ stats, int HW, int C, int G, float eps, int ncl) {
    pdl_ew_entry();
    const int b = blockIdx.x / ncl;
    const unsigned crank = ncl > 1 ? gn_cluster_rank() : 0u;
    const int cg = C / 8;             // 16
    const int g = threadIdx.x % cg;   // column group
    const int rl = threadIdx.x / cg;  // row lane
    const int rpb = 256 / cg;
    const int cpg = C / G;  // channels per group (4)
    const int rows = HW / ncl, r_begin = (int)crank * rows;  // this CTA's rows of the sample
    __shared__ float sm[2][256][8 + 1];
    __shared__ float gstat[64][2];
    __shared__ double part[64][2];  // this CTA's per-group partial sums (read remotely by the cluster peers)
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    const long base = (long)b * HW * cg;
    for (int r = r_begin + rl; r < r_begin + rows; r += rpb) {
        float v[8];
        load8(u_hi, u_lo, base + (long)r * cg + g, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s0[j] += v[j];
            s1[j] = fmaf(v[j], v[j], s1[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sm[0][threadIdx.x][j] = s0[j];
        sm[1][threadIdx.x][j] = s1[j];
    }
    __syncthreads();
    if (threadIdx.x < G) {
        const int grp = threadIdx.x;
        double a0 = 0, a1 = 0;
        for (int c = grp * cpg; c < (grp + 1) * cpg; ++c) {
            const int gg = c / 8, j = c % 8;
            for (int q = 0; q < rpb; ++q) {
                a0 += sm[0][q * cg + gg][j];
                a1 += sm[1][q * cg + gg][j];
            }
        }
        part[grp][0] = a0;
        part[grp][1] = a1;
    }
    if (ncl > 1) gn_cluster_sync(); else __syncthreads();
    if (threadIdx.x < G) {
        const int grp = threadIdx.x;
        double a0 = 0, a1 = 0;
        for (int r = 0; r < ncl; ++r) {  // fixed rank order: deterministic
            a0 += ncl > 1 ? gn_remote_f64(&part[grp][0], r) : part[grp][0];
            a1 += ncl > 1 ? gn_remote_f64(&part[grp][1], r) : part[grp][1];
        }
        const double n = (double)HW * cpg;
        const double m = a0 / n;
        double var = a1 / n - m * m;
        if (var < 0) var = 0;
        const float rstd = rsqrtf((float)var + eps);
        gstat[grp][0] = (float)m;
        gstat[grp][1] = rstd;
        if (crank == 0) {
            stats[((long)b * G + grp) * 2 + 0] = (float)m;
            stats[((long)b * G + grp) * 2 + 1] = rstd;
        }
    }
    __syncthreads();
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = g * 8 + j;
        const int grp = c / cpg;
        sc[j] = gamma[c] * gstat[grp][1];
        sh[j] = beta[c] - gstat[grp][0] * sc[j];
    }
    for (int r = r_begin + rl; r < r_begin + rows; r += rpb) {
        float v[8];
        const long off = base + (long)r * cg + g;
        load8(u_hi, u_lo, off, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(v[j], sc[j], sh[j]), 0.f);
        store8(y_hi, y_lo, off, v);
    }
    if (ncl > 1) gn_cluster_sync();  // no CTA may exit while a peer can still read its shared memory
}

// du = rstd * (dxh - mean_grp(dxh) - xh * mean_grp(dxh * xh)),  dxh = g*[y>0]*gamma;  dgamma += sum g*xh, dbeta += sum g
__global__ void __launch_bounds__(256) gn_relu_bwd_kernel(const bf16* __restrict__ g_hi, const bf16* __restrict__ g_lo,
                                                          const bf16* __restrict__ y_hi, const bf16* __restrict__ u_hi,
                                                          const bf16* __restrict__ u_lo, const float* __restrict__ gamma,
                                                          const float* __restrict__ stats, bf16* __restrict__ du_hi,
                                                          bf16* __restrict__ du_lo, float* __restrict__ dgamma,
                                                          float* __restrict__ dbeta, int HW, int C, int G, int ncl) {
    pdl_ew_entry();
    const int b = blockIdx.x / ncl;
    const unsigned crank = ncl > 1 ? gn_cluster_rank() : 0u;
    const int cg = C / 8;
    const int g = threadIdx.x % cg;
    const int rl = threadIdx.x / cg;
    const int rpb = 256 / cg;
    const int cpg = C / G;
    const int rows = HW / ncl, r_begin = (int)crank * rows;
    __shared__ float sm[2][256][8 + 1];
    __shared__ float gred[64][2];
    __shared__ double part[64][2];
    float mu[8], rs[8], ga[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = g * 8 + j;
        mu[j] = stats[((long)b * G + c / cpg) * 2 + 0];
        rs[j] = stats[((long)b * G + c / cpg) * 2 + 1];
        ga[j] = gamma[c];
    }
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    const long base = (long)b * HW * cg;
    for (int r = r_begin + rl; r < r_begin + rows; r += rpb) {
        const long off = base + (long)r * cg + g;
        float gv[8], y[8], u[8];
        load8(g_hi, g_lo, off, gv);
        unpack8(__ldg(reinterpret_cast<const uint4*>(y_hi) + off), y);
        load8(u_hi, u_lo, off, u);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float gg = y[j] > 0.f ? gv[j] : 0.f;
            const float xh = (u[j] - mu[j]) * rs[j];
            s0[j] += gg;
            s1[j] = fmaf(gg, xh, s1[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sm[0][threadIdx.x][j] = s0[j];
        sm[1][threadIdx.x][j] = s1[j];
    }
    __syncthreads();
    // per-channel sums -> dgamma/dbeta (atomics over samples / cluster ranks) and per-group sums of dxh, dxh*xh
    __shared__ float chs[2][128];
    for (int c = threadIdx.x; c < C; c += 256) {
        const int gg = c / 8, j = c % 8;
        float a0 = 0.f, a1 = 0.f;
        for (int q = 0; q < rpb; ++q) {
            a0 += sm[0][q * cg + gg][j];
            a1 += sm[1][q * cg + gg][j];
        }
        chs[0][c] = a0;
        chs[1][c] = a1;
        atomicAdd(dbeta + c, a0);
        atomicAdd(dgamma + c, a1);
    }
    __syncthreads();
    if (threadIdx.x < G) {
        const int grp = threadIdx.x;
        double a0 = 0, a1 = 0;
        for (int c = grp * cpg; c < (grp + 1) * cpg; ++c) {
            a0 += (double)chs[0][c] * gamma[c];
            a1 += (double)chs[1][c] * gamma[c];
        }
        part[grp][0] = a0;
        part[grp][1] = a1;
    }
    if (ncl > 1) gn_cluster_sync(); else __syncthreads();
    if (threadIdx.x < G) {
        const int grp = threadIdx.x;
        double a0 = 0, a1 = 0;
        for (int r = 0; r < ncl; ++r) {
            a0 += ncl > 1 ? gn_remote_f64(&part[grp][0], r) : part[grp][0];
            a1 += ncl > 1 ? gn_remote_f64(&part[grp][1], r) : part[grp][1];
        }
        const double n = (double)HW * cpg;
        gred[grp][0] = (float)(a0 / n);
        gred[grp][1] = (float)(a1 / n);
    }
    __syncthreads();
    for (int r = r_begin + rl; r < r_begin + rows; r += rpb) {
        const long off = base + (long)r * cg + g;
        float gv[8], y[8], u[8], o[8];
        load8(g_hi, g_lo, off, gv);
        unpack8(__ldg(reinterpret_cast<const uint4*>(y_hi) + off), y);
        load8(u_hi, u_lo, off, u);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int grp = (g * 8 + j) / cpg;
            const float gg = y[j] > 0.f ? gv[j] : 0.f;
            const float xh = (u[j] - mu[j]) * rs[j];
            o[j] = rs[j] * (gg * ga[j] - gred[grp][0] - xh * gred[grp][1]);
        }
        store8(du_hi, du_lo, off, o);
    }
    if (ncl > 1) gn_cluster_sync();
}

// out (bf16 hi/lo) = a + b   (gradient merge of two branches)
__global__ void add2_kernel(const bf16* __restrict__ a_hi, const bf16* __restrict__ a_lo, const bf16* __restrict__ b_hi,
                            const bf16* __restrict__ b_lo, bf16* __restrict__ o_hi, bf16* __restrict__ o_lo, long n8) {
    pdl_ew_entry();
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < n8; idx += (long)gridDim.x * blockDim.x) {
        float a[8], b[8];
        load8(a_hi, a_lo, idx, a);
        load8(b_hi, b_lo, idx, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += b[j];
        store8(o_hi, o_lo, idx, a);
    }
}

// fp32 [rows][C] -> bf16 hi/lo (and the reverse) for API-edge tensors
__global__ void f32_to_planes_kernel(const float* __restrict__ x, bf16* __restrict__ y_hi, bf16* __restrict__ y_lo, long n8) {
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < n8; idx += (long)gridDim.x * blockDim.x) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(x) + 2 * idx), b = __ldg(reinterpret_cast<const float4*>(x) + 2 * idx + 1);
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        store8(y_hi, y_lo, idx, v);
    }
}
__global__ void planes_to_f32_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo, float* __restrict__ y, long n8) {
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < n8; idx += (long)gridDim.x * blockDim.x) {
        float v[8];
        load8(x_hi, x_lo, idx, v);
        reinterpret_cast<float4*>(y)[2 * idx] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4*>(y)[2 * idx + 1] = make_float4(v[4], v[5], v[6], v[7]);
    }
}


// out[c] (+)= sum_rows x[r][c]   (bias gradients).  Block = 256 threads = (ld/8) column groups x row lanes.
__global__ void __launch_bounds__(256) colsum_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo,
                                                     float* __restrict__ out, long rows, int ld) {
    pdl_ew_entry();
    const int cg = ld / 8;
    const int rpb = 256 / cg;
    const int g = threadIdx.x % cg, rl = threadIdx.x / cg;
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = 0.f;
    if (rl < rpb) {
        for (long r = (long)blockIdx.x * rpb + rl; r < rows; r += (long)gridDim.x * rpb) {
            float v[8];
            load8(x_hi, x_lo, r * cg + g, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) s[j] += v[j];
        }
    }
    __shared__ float red[256][8 + 1];
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x][j] = s[j];
    __syncthreads();
    for (int c = threadIdx.x; c < ld; c += 256) {
        float a = 0.f;
        for (int q = 0; q < rpb; ++q) a += red[q * cg + c / 8][c % 8];
        atomicAdd(out + c, a);
    }
}

// LeakyReLU(0.1) backward through the saved OUTPUT y (sign(y) == sign(pre-activation)): g *= y > 0 ? 1 : 0.1
__global__ void leaky_bwd_kernel(const bf16* __restrict__ g_hi, const bf16* __restrict__ g_lo, const bf16* __restrict__ y_hi,
                                 bf16* __restrict__ o_hi, bf16* __restrict__ o_lo, long n8) {
    pdl_ew_entry();
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < n8; idx += (long)gridDim.x * blockDim.x) {
        float g[8], y[8];
        load8(g_hi, g_lo, idx, g);
        unpack8(__ldg(reinterpret_cast<const uint4*>(y_hi) + idx), y);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = y[j] > 0.f ? g[j] : 0.1f * g[j];
        store8(o_hi, o_lo, idx, g);
    }
}

// ------------------------------------------------------------------------------------------------
// GroupNorm(G, 256) + ReLU of the geometry head (ROT_HEAD.NORM = "GN"; cdpn_rot_head_region.py with get_norm("GN")), tensor
// [B][HW][256], HW in {256, 1024, 4096}.  Every reduction has a fixed decomposition and a fixed order, no atomics: the same
// inputs give bit-identical statistics and gradients on every run.  A crop is split into S = gn_head_splits(HW) slices of
// HW / S rows, one CTA per (slice, crop), so B = 4 already launches 128 CTAs at 64 x 64.
//   forward   stats_partial (per slice and group: sum x, sum x^2; fp32 per thread over <= 16 rows, double beyond) ->
//             stats_final (per crop and group, slices in order: mean, invstd) -> apply (relu(gamma x^ + beta) in fp32 before the
//             16-bit split, and the ReLU bitmap of the BatchNorm path: bit j of byte i = element 8 i + j > 0)
//   backward  bwd_partial (per slice and channel: sum dy, sum dy x^, dy masked by the bitmap) -> bwd_crop (per crop, slices in
//             order: the channel sums and the group means of gamma dy, gamma dy x^) -> bwd_param (dbeta, dgamma: crops in
//             order) -> bwd_apply (dx = invstd (gamma dy - mean(gamma dy) - x^ mean(gamma dy x^)))
// ------------------------------------------------------------------------------------------------
constexpr int kGnHeadC = 256;
constexpr int kGnHeadLanes = 8;  // row lanes per CTA: 256 threads = 32 column groups of 8 channels x 8 lanes

__host__ __device__ __forceinline__ int gn_head_splits(int HW) { return HW / 32 < 32 ? HW / 32 : 32; }

// workspace (doubles): forward partials [B][S][G][2]; backward partials [B][S][2][256] floats, then the crop sums
// [B][2][256] doubles, then the group means [B][G][2] floats
__host__ __device__ __forceinline__ long gn_head_ws_crop(int B, int S) { return (long)B * S * kGnHeadC; }
__host__ __device__ __forceinline__ long gn_head_ws_gred(int B, int S) { return gn_head_ws_crop(B, S) + (long)B * 2 * kGnHeadC; }

__global__ void __launch_bounds__(256) gn_head_stats_partial_kernel(const bf16* __restrict__ u_hi, const bf16* __restrict__ u_lo,
                                                                    double* __restrict__ part, int HW, int G) {
    const int s = blockIdx.x, S = gridDim.x, b = blockIdx.y;
    const int col = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int R = HW / S, cpg = kGnHeadC / G;
    __shared__ float red[2][kGnHeadLanes][kGnHeadC + 4];
    __shared__ double chs[2][kGnHeadC];
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    const long base = ((long)b * HW + (long)s * R) * 32 + col;
#pragma unroll 4
    for (int r = rl; r < R; r += kGnHeadLanes) {
        float v[8];
        load8(u_hi, u_lo, base + (long)r * 32, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s0[j] += v[j];
            s1[j] = fmaf(v[j], v[j], s1[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[0][rl][col * 8 + j] = s0[j];
        red[1][rl][col * 8 + j] = s1[j];
    }
    __syncthreads();
    {
        const int c = threadIdx.x;
        double a0 = 0.0, a1 = 0.0;
        for (int q = 0; q < kGnHeadLanes; ++q) {
            a0 += (double)red[0][q][c];
            a1 += (double)red[1][q][c];
        }
        chs[0][c] = a0;
        chs[1][c] = a1;
    }
    __syncthreads();
    if (threadIdx.x < 2 * G) {
        const int grp = threadIdx.x >> 1, k = threadIdx.x & 1;
        double a = 0.0;
        for (int c = grp * cpg; c < (grp + 1) * cpg; ++c) a += chs[k][c];
        part[(((long)b * S + s) * G + grp) * 2 + k] = a;
    }
}

__global__ void gn_head_stats_final_kernel(const double* __restrict__ part, float* __restrict__ stats, int B, int S, int G,
                                           double n, float eps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (crop, group)
    if (i >= B * G) return;
    const int b = i / G, grp = i % G;
    double a0 = 0.0, a1 = 0.0;
    for (int s = 0; s < S; ++s) {
        a0 += part[(((long)b * S + s) * G + grp) * 2 + 0];
        a1 += part[(((long)b * S + s) * G + grp) * 2 + 1];
    }
    const double m = a0 / n;
    double var = a1 / n - m * m;
    if (var < 0.0) var = 0.0;
    stats[(long)i * 2 + 0] = (float)m;
    stats[(long)i * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
}

// the per-channel (mean, invstd) of 8 consecutive channels c0.. of crop b: at most two groups (C / G >= 4)
__device__ __forceinline__ void gn_head_channel_stats(const float* __restrict__ stats, int b, int c0, int G, float (&mu)[8],
                                                      float (&rs)[8]) {
    const int cpg = kGnHeadC / G;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const long k = ((long)b * G + (c0 + j) / cpg) * 2;
        mu[j] = __ldg(stats + k);
        rs[j] = __ldg(stats + k + 1);
    }
}

__global__ void __launch_bounds__(256) gn_head_apply_kernel(const bf16* __restrict__ u_hi, const bf16* __restrict__ u_lo,
                                                            bf16* __restrict__ y_hi, bf16* __restrict__ y_lo,
                                                            uint8_t* __restrict__ mask_out, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, const float* __restrict__ stats,
                                                            long n8, int HW, int G) {
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < n8; idx += (long)gridDim.x * blockDim.x) {
        const int c0 = (int)(idx % 32) * 8;
        const int b = (int)(idx / 32 / HW);
        float v[8], mu[8], rs[8];
        load8(u_hi, u_lo, idx, v);
        gn_head_channel_stats(stats, b, c0, G, mu, rs);
        uint32_t bits = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float sc = __ldg(gamma + c0 + j) * rs[j];
            v[j] = fmaxf(fmaf(v[j], sc, fmaf(-mu[j], sc, __ldg(beta + c0 + j))), 0.f);
            bits |= (v[j] > 0.f ? 1u : 0u) << j;
        }
        store8(y_hi, y_lo, idx, v);
        if (mask_out != nullptr) mask_out[idx] = (uint8_t)bits;
    }
}

__global__ void __launch_bounds__(256) gn_head_bwd_partial_kernel(const bf16* __restrict__ g_hi, const bf16* __restrict__ g_lo,
                                                                  const bf16* __restrict__ u_hi, const bf16* __restrict__ u_lo,
                                                                  const uint8_t* __restrict__ mask_in,
                                                                  const float* __restrict__ stats, float* __restrict__ part,
                                                                  int HW, int G) {
    const int s = blockIdx.x, S = gridDim.x, b = blockIdx.y;
    const int col = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int R = HW / S;
    __shared__ float red[2][kGnHeadLanes][kGnHeadC + 4];
    float mu[8], rs[8], s0[8], s1[8];
    gn_head_channel_stats(stats, b, col * 8, G, mu, rs);
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    const long base = ((long)b * HW + (long)s * R) * 32 + col;
#pragma unroll 4
    for (int r = rl; r < R; r += kGnHeadLanes) {
        const long off = base + (long)r * 32;
        float gv[8], u[8];
        load8(g_hi, g_lo, off, gv);
        load8(u_hi, u_lo, off, u);
        const uint32_t bits = __ldg(mask_in + off);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float gg = ((bits >> j) & 1u) ? gv[j] : 0.f;
            s0[j] += gg;
            s1[j] = fmaf(gg, (u[j] - mu[j]) * rs[j], s1[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[0][rl][col * 8 + j] = s0[j];
        red[1][rl][col * 8 + j] = s1[j];
    }
    __syncthreads();
    const int c = threadIdx.x;
    float a0 = 0.f, a1 = 0.f;
    for (int q = 0; q < kGnHeadLanes; ++q) {
        a0 += red[0][q][c];
        a1 += red[1][q][c];
    }
    float* out = part + (((long)b * S + s) * 2) * kGnHeadC;
    out[c] = a0;
    out[kGnHeadC + c] = a1;
}

// one CTA per crop: channel sums over the slices (kept for the parameter gradients) and the group means of gamma dy, gamma dy x^
__global__ void __launch_bounds__(256) gn_head_bwd_crop_kernel(const float* __restrict__ part, const float* __restrict__ gamma,
                                                               double* __restrict__ crop, float* __restrict__ gred, int S, int G,
                                                               double n) {
    const int b = blockIdx.x, c = threadIdx.x, cpg = kGnHeadC / G;
    __shared__ double gs[2][kGnHeadC];
    double a0 = 0.0, a1 = 0.0;
    const float* p = part + (long)b * S * 2 * kGnHeadC + c;
    for (int s = 0; s < S; ++s) {
        a0 += (double)__ldg(p + (2L * s) * kGnHeadC);
        a1 += (double)__ldg(p + (2L * s + 1) * kGnHeadC);
    }
    crop[((long)b * 2) * kGnHeadC + c] = a0;
    crop[((long)b * 2 + 1) * kGnHeadC + c] = a1;
    const double ga = (double)__ldg(gamma + c);
    gs[0][c] = a0 * ga;
    gs[1][c] = a1 * ga;
    __syncthreads();
    if (threadIdx.x < 2 * G) {
        const int grp = threadIdx.x >> 1, k = threadIdx.x & 1;
        double a = 0.0;
        for (int q = grp * cpg; q < (grp + 1) * cpg; ++q) a += gs[k][q];
        gred[((long)b * G + grp) * 2 + k] = (float)(a / n);
    }
}

// dbeta[c] = sum over crops of sum dy, dgamma[c] = sum over crops of sum dy x^ (crops in order)
__global__ void __launch_bounds__(256) gn_head_bwd_param_kernel(const double* __restrict__ crop, float* __restrict__ dgamma,
                                                                float* __restrict__ dbeta, int B) {
    const int c = threadIdx.x, k = blockIdx.x;  // k = 0: dbeta, 1: dgamma
    double a = 0.0;
    for (int b = 0; b < B; ++b) a += crop[((long)b * 2 + k) * kGnHeadC + c];
    (k == 0 ? dbeta : dgamma)[c] = (float)a;
}

__global__ void __launch_bounds__(256) gn_head_bwd_apply_kernel(const bf16* __restrict__ g_hi, const bf16* __restrict__ g_lo,
                                                                const bf16* __restrict__ u_hi, const bf16* __restrict__ u_lo,
                                                                const uint8_t* __restrict__ mask_in, const float* __restrict__ gamma,
                                                                const float* __restrict__ stats, const float* __restrict__ gred,
                                                                bf16* __restrict__ du_hi, bf16* __restrict__ du_lo, long n8, int HW,
                                                                int G) {
    const int cpg = kGnHeadC / G;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < n8; idx += (long)gridDim.x * blockDim.x) {
        const int c0 = (int)(idx % 32) * 8;
        const int b = (int)(idx / 32 / HW);
        float gv[8], u[8], mu[8], rs[8], o[8];
        load8(g_hi, g_lo, idx, gv);
        load8(u_hi, u_lo, idx, u);
        const uint32_t bits = __ldg(mask_in + idx);
        gn_head_channel_stats(stats, b, c0, G, mu, rs);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const long k = ((long)b * G + (c0 + j) / cpg) * 2;
            const float gg = ((bits >> j) & 1u) ? gv[j] : 0.f;
            const float xh = (u[j] - mu[j]) * rs[j];
            o[j] = rs[j] * (fmaf(gg, __ldg(gamma + c0 + j), -__ldg(gred + k)) - xh * __ldg(gred + k + 1));
        }
        store8(du_hi, du_lo, idx, o);
    }
}

}  // namespace gdrn

using namespace gdrn;
#define STREAM cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_)
#define BF(p) reinterpret_cast<bf16*>(p)
#define CBF(p) reinterpret_cast<const bf16*>(p)
#define LAUNCH_DONE()                  \
    GDRN_CUDA_OK(cudaGetLastError()); \
    count_launch();                    \
    return 0

// GDRN_BN_REVERSE=0: BN forward / BN backward apply walk their tensors front to back like every other kernel (A/B; default: back
// to front, so that consecutive kernels of the chain meet in the part of a > L2 tensor that is still cached)
static int bn_reverse() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("GDRN_BN_REVERSE");
        v = e ? atoi(e) : 1;
    }
    return v;
}

extern "C" int gdrn_bn_finalize(const float* stats, const float* gamma, const float* beta, float* running_mean,
                                float* running_var, float* scale, float* shift, float* mean_out, float* invstd_out, int C,
                                float count, float eps, float momentum, int train, void* stream_) {
    STREAM;
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, stream>>>(stats, gamma, beta, running_mean, running_var, scale, shift,
                                                          mean_out, invstd_out, C, count, eps, momentum, train);
    LAUNCH_DONE();
}

extern "C" int gdrn_bn_fold_batched(const void* jobs_dev, int njobs, void* stream_) {
    STREAM;
    static_assert(sizeof(BnFoldJob) == 64, "BnFoldJob layout is mirrored by the host (gdr_net_b200/engine.py)");
    if (njobs <= 0) return 0;
    bn_fold_batched_kernel<<<dim3(njobs, 2), 256, 0, stream>>>(reinterpret_cast<const BnFoldJob*>(jobs_dev));
    LAUNCH_DONE();
}

extern "C" int gdrn_bn_act(const void* x_hi, const void* x_lo, const void* r_hi, const void* r_lo, void* y_hi, void* y_lo,
                           const float* scale, const float* shift, long rows, int C, int relu, void* stream_) {
    STREAM;
    if (C % 8) return set_error(GDRN_ERR_ARG, "bn_act: C %% 8 != 0");
    if (C > 512 || 256 % (C / 8)) return set_error(GDRN_ERR_ARG, "bn_act: unsupported C=%d", C);
    const int grid = ew_grid_amortised(rows * (C / 8), 256, 4);
#define GDRN_BN_ACT(LO, RES) \
    GDRN_LAUNCH_PDL_FWD((bn_act_kernel<LO, RES>), grid, 256, 0, stream, CBF(x_hi), CBF(x_lo), CBF(r_hi), CBF(r_lo), BF(y_hi), BF(y_lo), scale, shift, rows, C, relu)
    if (x_lo != nullptr) {
        if (r_hi != nullptr) GDRN_BN_ACT(true, true); else GDRN_BN_ACT(true, false);
    } else {
        if (r_hi != nullptr) GDRN_BN_ACT(false, true); else GDRN_BN_ACT(false, false);
    }
#undef GDRN_BN_ACT
    LAUNCH_DONE();
}

extern "C" int gdrn_maxpool_fwd(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, void* arg_out, int B, int H,
                                int W, int C, void* stream_) {
    STREAM;
    GDRN_LAUNCH_PDL_FWD(maxpool_fwd_kernel, ew_grid((long)B * (H / 2) * (W / 2) * (C / 8), 256), 256, 0, stream, 
        CBF(x_hi), CBF(x_lo), BF(y_hi), BF(y_lo), reinterpret_cast<uint8_t*>(arg_out), B, H, W, C);
    LAUNCH_DONE();
}
extern "C" int gdrn_maxpool_bwd(const void* arg_in, const void* g_hi, const void* g_lo, void* dx_hi, void* dx_lo, int B,
                                int H, int W, int C, void* stream_) {
    STREAM;
    GDRN_LAUNCH_PDL(maxpool_bwd_kernel, ew_grid((long)B * H * W * (C / 8), 256), 256, 0, stream, 
        reinterpret_cast<const uint8_t*>(arg_in), CBF(g_hi), CBF(g_lo), BF(dx_hi), BF(dx_lo), B, H, W, C);
    LAUNCH_DONE();
}
extern "C" int gdrn_upsample2x_fwd(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int B, int H, int W, int C,
                                   void* stream_) {
    STREAM;
    GDRN_LAUNCH_PDL_FWD(upsample2x_fwd_kernel, ew_grid((long)B * 4 * H * W * (C / 8), 256), 256, 0, stream, CBF(x_hi), CBF(x_lo), BF(y_hi),
                                                                                           BF(y_lo), B, H, W, C);
    LAUNCH_DONE();
}
extern "C" int gdrn_upsample2x_bwd(const void* g_hi, const void* g_lo, void* dx_hi, void* dx_lo, int B, int H, int W, int C,
                                   void* stream_) {
    STREAM;
    GDRN_LAUNCH_PDL(upsample2x_bwd_kernel, ew_grid((long)B * H * W * (C / 8), 256), 256, 0, stream, CBF(g_hi), CBF(g_lo), BF(dx_hi),
                                                                                       BF(dx_lo), B, H, W, C);
    LAUNCH_DONE();
}
extern "C" int gdrn_zero_insert(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int B, int H, int W, int C,
                                int mode, void* stream_) {
    STREAM;
    const long total = (long)B * H * W * (C / 8) * (mode == 0 ? 4 : 1);
    GDRN_LAUNCH_PDL_FWD(zero_insert_kernel, ew_grid(total, 256), 256, 0, stream, CBF(x_hi), CBF(x_lo), BF(y_hi), BF(y_lo), B, H, W, C, mode);
    LAUNCH_DONE();
}

extern "C" int gdrn_bn_bwd(const void* ga_hi, const void* ga_lo, const void* gb_hi, const void* gb_lo, const void* y_hi,
                           const void* u_hi, const void* u_lo, const float* mean, const float* invstd, const float* gamma,
                           const float* beta, float* sums, void* du_hi, void* du_lo, void* gout_hi, void* gout_lo,
                           float* dgamma, float* dbeta, const void* relu_mask, float* det_ws, long rows, int C, int train,
                           int flags, void* stream_) {
    STREAM;
    const uint8_t* mask_in = reinterpret_cast<const uint8_t*>(relu_mask);
    const bool det = (flags & 4) != 0;
    if (det && det_ws == nullptr) return set_error(GDRN_ERR_ARG, "bn_bwd: deterministic mode needs a workspace of 2*C*%d floats", 2 * num_sms());
    if (C % 64 || C > 512) return set_error(GDRN_ERR_ARG, "bn_bwd: unsupported C=%d", C);
    const int mask_u = flags & 1;
    if (mask_u && (y_hi != nullptr || beta == nullptr)) return set_error(GDRN_ERR_ARG, "bn_bwd: mask-from-u needs beta and no y");
    {  // the reductions also provide dgamma / dbeta when BN runs on frozen (eval) statistics
        if (!(flags & 2) && !det) GDRN_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(float) * 2 * C, stream));
        const int rpb = kBnBwdThreads / (C / 8);
        long blocks = (rows + (long)rpb * 16 - 1) / ((long)rpb * 16);  // >= 16 rows per thread: few atomics, amortised prologue
        const long cap = (long)num_sms() * 2;
        if (blocks > cap) blocks = cap;
        if (blocks < 1) blocks = 1;
#define GDRN_BN_RED(LO, MU)                                                                                                   \
    GDRN_LAUNCH_PDL((bn_bwd_reduce_kernel<LO, MU>), (int)blocks, kBnBwdThreads, 0, stream, CBF(ga_hi), CBF(ga_lo), CBF(gb_hi), CBF(gb_lo),       \
                                                                            CBF(y_hi), CBF(u_hi), CBF(u_lo), mean, invstd, gamma, \
                                                                            beta, sums, rows, C, mask_in, det ? det_ws : nullptr)
        if (u_lo != nullptr) {
            if (mask_u) GDRN_BN_RED(true, true); else GDRN_BN_RED(true, false);
        } else {
            if (mask_u) GDRN_BN_RED(false, true); else GDRN_BN_RED(false, false);
        }
#undef GDRN_BN_RED
        GDRN_CUDA_OK(cudaGetLastError());
        count_launch();
        if (det) {
            sum_partials_kernel<<<(2 * C + 255) / 256, 256, 0, stream>>>(det_ws, (int)blocks, 2 * C, sums);
            GDRN_CUDA_OK(cudaGetLastError());
            count_launch();
        }
    }
    const int agrid = ew_grid_amortised(rows * (C / 8), 256, 4);
#define GDRN_BN_APP(LO, MU)                                                                                                      \
    GDRN_LAUNCH_PDL((bn_bwd_apply_kernel<LO, MU>), agrid, 256, 0, stream, CBF(ga_hi), CBF(ga_lo), CBF(gb_hi), CBF(gb_lo), CBF(y_hi), CBF(u_hi),    \
                                                           CBF(u_lo), mean, invstd, gamma, beta, sums, BF(du_hi), BF(du_lo),       \
                                                           BF(gout_hi), BF(gout_lo), dgamma, dbeta, rows, C, train, mask_in, bn_reverse())
    if (u_lo != nullptr) {
        if (mask_u) GDRN_BN_APP(true, true); else GDRN_BN_APP(true, false);
    } else {
        if (mask_u) GDRN_BN_APP(false, true); else GDRN_BN_APP(false, false);
    }
#undef GDRN_BN_APP
    LAUNCH_DONE();
}

// deterministic BatchNorm batch statistics straight from the tensor (two-stage, ordered): stats[0][c] = sum, stats[1][c] = sum of
// squares.  ws: >= 2 * C * gdrn_det_parts() floats.
extern "C" int gdrn_det_parts() { return 2 * num_sms(); }
extern "C" int gdrn_bn_stats(const void* u_hi, const void* u_lo, float* ws, float* stats, long rows, int C, void* stream_) {
    STREAM;
    if (C % 64 || C > 512) return set_error(GDRN_ERR_ARG, "bn_stats: unsupported C=%d", C);
    const int rpb = kBnBwdThreads / (C / 8);
    long blocks = (rows + (long)rpb * 16 - 1) / ((long)rpb * 16);
    const long cap = (long)num_sms() * 2;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (u_lo != nullptr) bn_stats_partial_kernel<true><<<(int)blocks, kBnBwdThreads, 0, stream>>>(CBF(u_hi), CBF(u_lo), ws, rows, C);
    else bn_stats_partial_kernel<false><<<(int)blocks, kBnBwdThreads, 0, stream>>>(CBF(u_hi), CBF(u_lo), ws, rows, C);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    sum_partials_kernel<<<(2 * C + 255) / 256, 256, 0, stream>>>(ws, (int)blocks, 2 * C, stats);
    LAUNCH_DONE();
}

extern "C" int gdrn_gn_relu_fwd(const void* u_hi, const void* u_lo, void* y_hi, void* y_lo, const float* gamma,
                                const float* beta, float* stats, int B, int HW, int C, int G, float eps, void* stream_) {
    STREAM;
    if (C != 128 || G > 64 || C % G) return set_error(GDRN_ERR_ARG, "gn_relu_fwd: only C=128 supported");
    const int ncl = (HW % (kGnCluster * 16) == 0) ? kGnCluster : 1;  // a sample's rows split over a cluster of CTAs (DSMEM exchange)
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(B * ncl);
    cfg.blockDim = dim3(256);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = ncl;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    GDRN_CUDA_OK(cudaLaunchKernelEx(&cfg, gn_relu_fwd_kernel, CBF(u_hi), CBF(u_lo), BF(y_hi), BF(y_lo), gamma, beta, stats, HW, C, G, eps, ncl));
    count_launch();
    return 0;
}
extern "C" int gdrn_gn_relu_bwd(const void* g_hi, const void* g_lo, const void* y_hi, const void* u_hi, const void* u_lo,
                                const float* gamma, const float* stats, void* du_hi, void* du_lo, float* dgamma,
                                float* dbeta, int B, int HW, int C, int G, void* stream_) {
    STREAM;
    if (C != 128 || G > 64 || C % G) return set_error(GDRN_ERR_ARG, "gn_relu_bwd: only C=128 supported");
    const int ncl = (HW % (kGnCluster * 16) == 0) ? kGnCluster : 1;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(B * ncl);
    cfg.blockDim = dim3(256);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = ncl;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    GDRN_CUDA_OK(cudaLaunchKernelEx(&cfg, gn_relu_bwd_kernel, CBF(g_hi), CBF(g_lo), CBF(y_hi), CBF(u_hi), CBF(u_lo), gamma, stats,
                                    BF(du_hi), BF(du_lo), dgamma, dbeta, HW, C, G, ncl));
    count_launch();
    return 0;
}
extern "C" int gdrn_add2(const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo, void* o_hi, void* o_lo,
                         long n, void* stream_) {
    STREAM;
    GDRN_LAUNCH_PDL(add2_kernel, ew_grid(n / 8, 256), 256, 0, stream, CBF(a_hi), CBF(a_lo), CBF(b_hi), CBF(b_lo), BF(o_hi), BF(o_lo), n / 8);
    LAUNCH_DONE();
}
extern "C" int gdrn_f32_to_planes(const float* x, void* y_hi, void* y_lo, long n, void* stream_) {
    STREAM;
    f32_to_planes_kernel<<<ew_grid(n / 8, 256), 256, 0, stream>>>(x, BF(y_hi), BF(y_lo), n / 8);
    LAUNCH_DONE();
}
extern "C" int gdrn_planes_to_f32(const void* x_hi, const void* x_lo, float* y, long n, void* stream_) {
    STREAM;
    planes_to_f32_kernel<<<ew_grid(n / 8, 256), 256, 0, stream>>>(CBF(x_hi), CBF(x_lo), y, n / 8);
    LAUNCH_DONE();
}

extern "C" int gdrn_colsum(const void* x_hi, const void* x_lo, float* out, long rows, int ld, void* stream_) {
    STREAM;
    if (ld % 8 || ld / 8 > 256 || 256 % (ld / 8)) return set_error(GDRN_ERR_ARG, "colsum: unsupported ld=%d", ld);
    GDRN_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * ld, stream));
    const int rpb = 256 / (ld / 8);
    long blocks = (rows + rpb - 1) / rpb;
    const long cap = (long)num_sms() * 4;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    GDRN_LAUNCH_PDL(colsum_kernel, (int)blocks, 256, 0, stream, CBF(x_hi), CBF(x_lo), out, rows, ld);
    LAUNCH_DONE();
}
extern "C" int gdrn_leaky_bwd(const void* g_hi, const void* g_lo, const void* y_hi, void* o_hi, void* o_lo, long n,
                              void* stream_) {
    STREAM;
    GDRN_LAUNCH_PDL(leaky_bwd_kernel, ew_grid(n / 8, 256), 256, 0, stream, CBF(g_hi), CBF(g_lo), CBF(y_hi), BF(o_hi), BF(o_lo), n / 8);
    LAUNCH_DONE();
}

extern "C" int gdrn_bn_fwd(const void* x_hi, const void* x_lo, const void* r_hi, const void* r_lo, void* y_hi, void* y_lo,
                           const float* stats, const float* gamma, const float* beta, float* running_mean, float* running_var,
                           float* mean_out, float* invstd_out, void* relu_mask_out, long rows, int C, float eps, float momentum,
                           int train, int relu, void* stream_) {
    STREAM;
    if (C % 8 || C > 512 || 256 % (C / 8)) return set_error(GDRN_ERR_ARG, "bn_fwd: unsupported C=%d", C);
    if (train && stats == nullptr) return set_error(GDRN_ERR_ARG, "bn_fwd: batch statistics missing");
    const int grid = ew_grid_amortised(rows * (C / 8), 256, 4);
#define GDRN_BN_FWD(LO, RES)                                                                                                  \
    GDRN_LAUNCH_PDL_FWD((bn_fwd_kernel<LO, RES>), grid, 256, 0, stream, CBF(x_hi), CBF(x_lo), CBF(r_hi), CBF(r_lo), BF(y_hi), BF(y_lo), stats, gamma, beta, \
                                                     running_mean, running_var, mean_out, invstd_out, rows, C, eps, momentum, train, relu,  \
                                                     reinterpret_cast<uint8_t*>(relu_mask_out), bn_reverse())
    if (x_lo != nullptr) {
        if (r_hi != nullptr) GDRN_BN_FWD(true, true); else GDRN_BN_FWD(true, false);
    } else {
        if (r_hi != nullptr) GDRN_BN_FWD(false, true); else GDRN_BN_FWD(false, false);
    }
#undef GDRN_BN_FWD
    LAUNCH_DONE();
}

static int check_head_gn(const char* fn, int B, int HW, int C, int G) {
    if (C != kGnHeadC) return set_error(GDRN_ERR_ARG, "%s: C = %d (the geometry head's GroupNorm has C = 256)", fn, C);
    if (G < 1 || G > 64 || kGnHeadC % G) return set_error(GDRN_ERR_ARG, "%s: G = %d (a divisor of 256, at most 64)", fn, G);
    if (HW != 256 && HW != 1024 && HW != 4096) return set_error(GDRN_ERR_ARG, "%s: HW = %d (256, 1024 or 4096)", fn, HW);
    if (B < 1) return set_error(GDRN_ERR_ARG, "%s: B = %d", fn, B);
    return 0;
}

extern "C" long long gdrn_head_gn_workspace(int B, int HW) {
    if (B < 1 || (HW != 256 && HW != 1024 && HW != 4096)) return -1;
    return gn_head_ws_gred(B, gn_head_splits(HW)) + (long long)B * 64;
}

extern "C" int gdrn_head_gn_fwd(const void* u_hi, const void* u_lo, void* y_hi, void* y_lo, void* relu_mask_out, const float* gamma,
                                const float* beta, float* stats, double* ws, int B, int HW, int C, int G, float eps, void* stream_) {
    STREAM;
    if (int rc = check_head_gn("head_gn_fwd", B, HW, C, G)) return rc;
    if (!u_hi || !y_hi || !gamma || !beta || !stats || !ws)
        return set_error(GDRN_ERR_ARG, "head_gn_fwd: u, y, gamma, beta, stats and the workspace are required");
    const int S = gn_head_splits(HW);
    gn_head_stats_partial_kernel<<<dim3(S, B), 256, 0, stream>>>(CBF(u_hi), CBF(u_lo), ws, HW, G);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    gn_head_stats_final_kernel<<<(B * G + 127) / 128, 128, 0, stream>>>(ws, stats, B, S, G, (double)HW * (kGnHeadC / G), eps);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    const long n8 = (long)B * HW * (kGnHeadC / 8);
    gn_head_apply_kernel<<<ew_grid(n8, 256), 256, 0, stream>>>(CBF(u_hi), CBF(u_lo), BF(y_hi), BF(y_lo),
                                                               reinterpret_cast<uint8_t*>(relu_mask_out), gamma, beta, stats, n8, HW, G);
    LAUNCH_DONE();
}

extern "C" int gdrn_head_gn_bwd(const void* g_hi, const void* g_lo, const void* u_hi, const void* u_lo, const void* relu_mask,
                                const float* gamma, const float* stats, void* du_hi, void* du_lo, float* dgamma, float* dbeta,
                                double* ws, int B, int HW, int C, int G, void* stream_) {
    STREAM;
    if (int rc = check_head_gn("head_gn_bwd", B, HW, C, G)) return rc;
    if (!g_hi || !u_hi || !relu_mask || !gamma || !stats || !du_hi || !dgamma || !dbeta || !ws)
        return set_error(GDRN_ERR_ARG, "head_gn_bwd: g, u, the ReLU mask, gamma, stats, du, dgamma, dbeta and the workspace are required");
    const int S = gn_head_splits(HW);
    float* part = reinterpret_cast<float*>(ws);
    double* crop = ws + gn_head_ws_crop(B, S);
    float* gred = reinterpret_cast<float*>(ws + gn_head_ws_gred(B, S));
    const uint8_t* mask = reinterpret_cast<const uint8_t*>(relu_mask);
    gn_head_bwd_partial_kernel<<<dim3(S, B), 256, 0, stream>>>(CBF(g_hi), CBF(g_lo), CBF(u_hi), CBF(u_lo), mask, stats, part, HW, G);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    gn_head_bwd_crop_kernel<<<B, 256, 0, stream>>>(part, gamma, crop, gred, S, G, (double)HW * (kGnHeadC / G));
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    gn_head_bwd_param_kernel<<<2, 256, 0, stream>>>(crop, dgamma, dbeta, B);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    const long n8 = (long)B * HW * (kGnHeadC / 8);
    gn_head_bwd_apply_kernel<<<ew_grid(n8, 256), 256, 0, stream>>>(CBF(g_hi), CBF(g_lo), CBF(u_hi), CBF(u_lo), mask, gamma, stats,
                                                                   gred, BF(du_hi), BF(du_lo), n8, HW, G);
    LAUNCH_DONE();
}
