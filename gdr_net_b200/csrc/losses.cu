// Geometry glue, per-pixel losses and pose decode / point-matching loss of the GDR-Net hot path.
//
//   head_glue_fwd   GDRN.py:156-169 + conv_pnp_net.py:120-125: softmax(region[:,1:]), cat(xyz, coord2d, region),
//                   (xyz-0.5)*extent  -> NHWC bf16 Patch-PnP input (69 valid of 128 channels)
//   pixel_loss_fwd  GDRN.py:341-400: masked L1 on x,y,z, L1 / BCE / 2-class CE mean on mask, CE-sum on region (SURVEY P5
//                   quirk); each of the three takes its own GT mask (XYZ_LOSS_MASK_GT, MASK_LOSS_GT, REGION_LOSS_MASK_GT)
//   head_bwd        analytic backward of both of the above, fused: one pass over the logits
//   pose_loss       rot_reps.py:34-49, pose_from_pred_centroid_z.py:144-227, utils.py:208-236,
//                   pose_utils.py:323-370 (quat2mat), pm_loss.py:82-114, pose_utils.py:430-482 (closest
//                   symmetric GT, on device instead of the reference's host loop), GDRN.py:439-471,
//                   model_utils.py:40-52 (mean re / te logging) -- forward + analytic/forward-mode backward.
#include <math.h>

#include "../../include/gdrn_b200.h"
#include "gdrn_internal.h"
#include "ptx.cuh"
#include "pixel_head.cuh"

namespace gdrn {

// ------------------------------------------------------------------------------------------------
// W2D: the Patch-PnP input carries the 2-D crop coordinates (cfg PNP_NET.WITH_2D_COORD: 3 + 2 + 64 = 69 channels, region at
// 5..68) or not (3 + 64 = 67 channels, region at 3..66) -- GDRN.py:171-173, :635-647
template <int MO, bool W2D>
__global__ void __launch_bounds__(128) head_glue_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ coord2d,
                                                            const float* __restrict__ extents, bf16* __restrict__ out_hi,
                                                            bf16* __restrict__ out_lo, int B, int HW) {
    const long total = (long)B * HW;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < total; pix += (long)gridDim.x * blockDim.x) {
        const int b = (int)(pix / HW);
        const int hw = (int)(pix - (long)b * HW);
        float z[kLogitLd];
        load_logits(logits, pix, z);
        float o[72];
#pragma unroll
        for (int j = 0; j < 3; ++j) o[j] = (z[MO + j] - 0.5f) * __ldg(extents + b * 3 + j);
        constexpr int RO = W2D ? 5 : 3;  // first region channel
        if (W2D) {
            o[3] = __ldg(coord2d + ((long)b * 2 + 0) * HW + hw);
            o[4] = __ldg(coord2d + ((long)b * 2 + 1) * HW + hw);
        }
        float m = -INFINITY;
#pragma unroll
        for (int k = 0; k < kNumReg; ++k) m = fmaxf(m, z[MO + 4 + k]);
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kNumReg; ++k) {
            o[RO + k] = expf(z[MO + 4 + k] - m);
            s += o[RO + k];
        }
        const float inv = 1.f / s;
#pragma unroll
        for (int k = 0; k < kNumReg; ++k) o[RO + k] *= inv;
#pragma unroll
        for (int k = RO + kNumReg; k < 72; ++k) o[k] = 0.f;
        store_row_bf16(out_hi, out_lo, pix, kPnpLd, o, 72);
        // zero the padding channels 72..127
        const uint4 zz = make_uint4(0, 0, 0, 0);
        for (int j = 72; j < kPnpLd; j += 8) {
            *reinterpret_cast<uint4*>(out_hi + pix * kPnpLd + j) = zz;
            if (out_lo != nullptr) *reinterpret_cast<uint4*>(out_lo + pix * kPnpLd + j) = zz;
        }
    }
}

// Patch-PnP input packing for the STANDALONE ConvPnPNet.forward (conv_pnp_net.py:111-125): coor_feat [B][c_feat][HW] fp32
// (xyz [+ 2-D coords]) and region [B][c_reg][HW] fp32 (NCHW, the reference's layout) -> NHWC 16-bit planes [B*HW][128];
// xyz is de-normalised by the extents when c_feat is 3 or 5 (:120-122).  One thread per pixel: the per-channel reads are
// coalesced across the warp (consecutive pixels), each thread emits its pixel's 256-byte row.
__global__ void __launch_bounds__(128) pnp_pack_input_kernel(const float* __restrict__ coor, int c_feat,
                                                             const float* __restrict__ region, int c_reg,
                                                             const float* __restrict__ extents, bf16* __restrict__ out_hi,
                                                             bf16* __restrict__ out_lo, int B, int HW) {
    const long total = (long)B * HW;
    const bool denorm = (c_feat == 3 || c_feat == 5) && extents != nullptr;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < total; pix += (long)gridDim.x * blockDim.x) {
        const int b = (int)(pix / HW);
        const int hw = (int)(pix - (long)b * HW);
        float o[72];
#pragma unroll
        for (int k = 0; k < 72; ++k) {
            float v = 0.f;
            if (k < c_feat) {
                v = __ldg(coor + ((long)b * c_feat + k) * HW + hw);
                if (denorm && k < 3) v = (v - 0.5f) * __ldg(extents + b * 3 + k);
            } else if (k < c_feat + c_reg) {
                v = __ldg(region + ((long)b * c_reg + (k - c_feat)) * HW + hw);
            }
            o[k] = v;
        }
        store_row_bf16(out_hi, out_lo, pix, kPnpLd, o, 72);
        const uint4 zz = make_uint4(0, 0, 0, 0);
        for (int j = 72; j < kPnpLd; j += 8) {
            *reinterpret_cast<uint4*>(out_hi + pix * kPnpLd + j) = zz;
            if (out_lo != nullptr) *reinterpret_cast<uint4*>(out_lo + pix * kPnpLd + j) = zz;
        }
    }
}

// sums (double[7]): |dx|, |dy|, |dz| (masked), mask loss, region CE, sum(xyz mask), sum(region mask).  SEP = the region mask
// is not the xyz mask; without it the region terms reuse the xyz mask and slot 6 gets slot 5's partials.  n_sums = 6 writes
// slots 0..5 only (the original six-slot layout; needs !SEP).
template <int MODE, int MO, bool SEP>
__global__ void __launch_bounds__(128) pixel_loss_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ gt_xyz,
                                                             const float* __restrict__ m_xyz, const float* __restrict__ m_tgt,
                                                             const float* __restrict__ m_reg, const long long* __restrict__ labels,
                                                             double* __restrict__ sums, int n_sums, int B, int HW) {
    constexpr int NACC = SEP ? 7 : 6;
    const long total = (long)B * HW;
    float acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) acc[j] = 0.f;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < total; pix += (long)gridDim.x * blockDim.x) {
        const int b = (int)(pix / HW);
        const int hw = (int)(pix - (long)b * HW);
        float z[kLogitLd];
        load_logits(logits, pix, z);
        const float mv = __ldg(m_xyz + pix), mt = __ldg(m_tgt + pix);
        const float mr = SEP ? __ldg(m_reg + pix) : mv;
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[j] += fabsf(masked_diff(z[MO + j], __ldg(gt_xyz + ((long)b * 3 + j) * HW + hw), mv));
        acc[3] += mask_loss<MODE>(z, mt);
        // CE over 65 logits (bg + 64), logits and label multiplied by the region mask
        float mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < 65; ++k) mx = fmaxf(mx, z[MO + 3 + k] * mr);
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 65; ++k) s += expf(z[MO + 3 + k] * mr - mx);
        const int lab = (int)(__ldg(labels + pix) * (long long)mr);
        float zl = 0.f;
#pragma unroll
        for (int k = 0; k < 65; ++k) zl = (k == lab) ? z[MO + 3 + k] * mr : zl;
        acc[4] += (logf(s) + mx) - zl;
        acc[5] += mv;
        if (SEP) acc[NACC - 1] += mr;
    }
    __shared__ float red[NACC][4];
#pragma unroll
    for (int j = 0; j < NACC; ++j) {
        float v = acc[j];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[j][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x < n_sums) {
        const int j = threadIdx.x < NACC ? threadIdx.x : 5;
        const float v = red[j][0] + red[j][1] + red[j][2] + red[j][3];
        atomicAdd(sums + threadIdx.x, (double)v);
    }
}

// d_logits (bf16 hi/lo, [P][128], cols >= 68 + MO zero) = d(pixel losses) + glue backward of d_pnp_in
// gw[5]: upstream gradients of loss_coor_x, _y, _z, loss_mask, loss_region.  Normalisers: sums[5] (xyz), sums[6] (region, SEP
// only: without SEP the region mask is the xyz mask and slot 6 is not read).
template <int MODE, int MO, bool SEP, bool W2D>
__global__ void __launch_bounds__(128) head_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ gt_xyz,
                                                       const float* __restrict__ m_xyz, const float* __restrict__ m_tgt,
                                                       const float* __restrict__ m_reg, const long long* __restrict__ labels,
                                                       const double* __restrict__ sums,
                                                       const float* __restrict__ gw, const bf16* __restrict__ din_hi,
                                                       const bf16* __restrict__ din_lo, const float* __restrict__ extents,
                                                       bf16* __restrict__ out_hi, bf16* __restrict__ out_lo, int B, int HW) {
    const long total = (long)B * HW;
    const float inv_fg = 1.f / fmaxf((float)sums[5], 1.f);
    const float inv_reg = SEP ? 1.f / fmaxf((float)sums[6], 1.f) : inv_fg;
    const float inv_all = 1.f / (float)total;
    const float gwx = gw[0], gwy = gw[1], gwz = gw[2], gwm = gw[3], gwr = gw[4];
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < total; pix += (long)gridDim.x * blockDim.x) {
        const int b = (int)(pix / HW);
        const int hw = (int)(pix - (long)b * HW);
        float z[kLogitLd];
        load_logits(logits, pix, z);
        const float mv = __ldg(m_xyz + pix), mt = __ldg(m_tgt + pix);
        const float mr = SEP ? __ldg(m_reg + pix) : mv;
        float d[72];
        // mask channels: mean over B HW pixels
        mask_loss_bwd<MODE>(z, mt, gwm * inv_all, d);
        // Patch-PnP input gradient (hi+lo)
        float gin[72];
        if (din_hi != nullptr) {
            for (int j = 0; j < 72; j += 8) {
                const uint4 q = __ldg(reinterpret_cast<const uint4*>(din_hi + pix * kPnpLd + j));
                const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    unpack_hi2(w[t], gin[j + 2 * t], gin[j + 2 * t + 1]);
                }
                if (din_lo != nullptr) {
                    const uint4 q2 = __ldg(reinterpret_cast<const uint4*>(din_lo + pix * kPnpLd + j));
                    const uint32_t w2[4] = {q2.x, q2.y, q2.z, q2.w};
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        float ra, rb;
                        unpack_lo2(w2[t], ra, rb);
                        gin[j + 2 * t] += ra;
                        gin[j + 2 * t + 1] += rb;
                    }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 72; ++j) gin[j] = 0.f;
        }
        // xyz channels
        const float gws[3] = {gwx, gwy, gwz};
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float e = masked_diff(z[MO + j], __ldg(gt_xyz + ((long)b * 3 + j) * HW + hw), mv);
            const float sg = e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f);
            d[MO + j] = gws[j] * inv_fg * sg * mv + gin[j] * __ldg(extents + b * 3 + j);
        }
        // region CE over 65 (masked logits): d = m * (softmax65(z*m) - onehot(label*m)) / max(sum m, 1)
        {
            float mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < 65; ++k) mx = fmaxf(mx, z[MO + 3 + k] * mr);
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 65; ++k) {
                d[MO + 3 + k] = expf(z[MO + 3 + k] * mr - mx);
                s += d[MO + 3 + k];
            }
            const float c = gwr * inv_reg * mr;
            const float inv = 1.f / s;
            const int lab = (int)(__ldg(labels + pix) * (long long)mr);
#pragma unroll
            for (int k = 0; k < 65; ++k) d[MO + 3 + k] = c * (d[MO + 3 + k] * inv - (k == lab ? 1.f : 0.f));
        }
        // softmax64 backward of the Patch-PnP region-attention input: dz_k = p_k (g_k - sum_j g_j p_j)
        if (din_hi != nullptr) {
            constexpr int RO = W2D ? 5 : 3;  // first region channel of the Patch-PnP input
            float mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) mx = fmaxf(mx, z[MO + 4 + k]);
            float s = 0.f, dot = 0.f;
            float pk[kNumReg];
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) {
                pk[k] = expf(z[MO + 4 + k] - mx);
                s += pk[k];
            }
            const float inv = 1.f / s;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) {
                pk[k] *= inv;
                dot = fmaf(gin[RO + k], pk[k], dot);
            }
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) d[MO + 4 + k] += pk[k] * (gin[RO + k] - dot);
        }
#pragma unroll
        for (int k = 68 + MO; k < 72; ++k) d[k] = 0.f;
        store_row_bf16(out_hi, out_lo, pix, kPnpLd, d, 72);
        const uint4 zz = make_uint4(0, 0, 0, 0);
        for (int j = 72; j < kPnpLd; j += 8) {
            *reinterpret_cast<uint4*>(out_hi + pix * kPnpLd + j) = zz;
            if (out_lo != nullptr) *reinterpret_cast<uint4*>(out_lo + pix * kPnpLd + j) = zz;
        }
    }
}

// pixel_loss_fwd_kernel with the region CE over R + 1 classes (bg + nreg regions)
template <int MODE, int MO, bool SEP>
__global__ void __launch_bounds__(128) pixel_loss_fwd2_kernel(const float* __restrict__ logits, const float* __restrict__ gt_xyz,
                                                              const float* __restrict__ m_xyz, const float* __restrict__ m_tgt,
                                                              const float* __restrict__ m_reg, const long long* __restrict__ labels,
                                                              double* __restrict__ sums, int B, int HW, int nreg) {
    constexpr int NACC = SEP ? 7 : 6;
    const long total = (long)B * HW;
    float acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) acc[j] = 0.f;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < total; pix += (long)gridDim.x * blockDim.x) {
        const int b = (int)(pix / HW);
        const int hw = (int)(pix - (long)b * HW);
        float z[kLogitLd];
        load_logits(logits, pix, z);
        const float mv = __ldg(m_xyz + pix), mt = __ldg(m_tgt + pix);
        const float mr = SEP ? __ldg(m_reg + pix) : mv;
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[j] += fabsf(masked_diff(z[MO + j], __ldg(gt_xyz + ((long)b * 3 + j) * HW + hw), mv));
        acc[3] += mask_loss<MODE>(z, mt);
        // CE over nreg + 1 logits, logits and label multiplied by the region mask
        float mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < 65; ++k) mx = k <= nreg ? fmaxf(mx, z[MO + 3 + k] * mr) : mx;
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 65; ++k) s += k <= nreg ? expf(z[MO + 3 + k] * mr - mx) : 0.f;
        const int lab = (int)(__ldg(labels + pix) * (long long)mr);
        float zl = 0.f;
#pragma unroll
        for (int k = 0; k < 65; ++k) zl = (k == lab && k <= nreg) ? z[MO + 3 + k] * mr : zl;
        acc[4] += (logf(s) + mx) - zl;
        acc[5] += mv;
        if (SEP) acc[NACC - 1] += mr;
    }
    __shared__ float red[NACC][4];
#pragma unroll
    for (int j = 0; j < NACC; ++j) {
        float v = acc[j];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[j][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        const int j = threadIdx.x < NACC ? threadIdx.x : 5;
        const float v = red[j][0] + red[j][1] + red[j][2] + red[j][3];
        atomicAdd(sums + threadIdx.x, (double)v);
    }
}

// ------------------------------------------------------------------------------------------------
// Forward-mode dual numbers with 9 tangents (d/d rot6d[0..5], d/d t[0..2])
// ------------------------------------------------------------------------------------------------
struct Dual {
    float v;
    float d[9];
};
__device__ __forceinline__ Dual dconst(float c) {
    Dual r;
    r.v = c;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = 0.f;
    return r;
}
__device__ __forceinline__ Dual dvar(float c, int idx) {
    Dual r = dconst(c);
    r.d[idx] = 1.f;
    return r;
}
__device__ __forceinline__ Dual operator+(const Dual& a, const Dual& b) {
    Dual r;
    r.v = a.v + b.v;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] + b.d[i];
    return r;
}
__device__ __forceinline__ Dual operator-(const Dual& a, const Dual& b) {
    Dual r;
    r.v = a.v - b.v;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] - b.d[i];
    return r;
}
__device__ __forceinline__ Dual operator-(const Dual& a) {
    Dual r;
    r.v = -a.v;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = -a.d[i];
    return r;
}
__device__ __forceinline__ Dual operator*(const Dual& a, const Dual& b) {
    Dual r;
    r.v = a.v * b.v;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
    return r;
}
__device__ __forceinline__ Dual operator*(const Dual& a, float s) {
    Dual r;
    r.v = a.v * s;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] * s;
    return r;
}
__device__ __forceinline__ Dual operator/(const Dual& a, const Dual& b) {
    Dual r;
    const float inv = 1.f / b.v;
    r.v = a.v * inv;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv;
    return r;
}
__device__ __forceinline__ Dual dsqrt(const Dual& a) {
    Dual r;
    r.v = sqrtf(a.v);
    const float k = a.v > 0.f ? 0.5f / r.v : 0.f;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] * k;
    return r;
}
__device__ __forceinline__ Dual dacos(const Dual& a) {
    Dual r;
    r.v = acosf(a.v);
    const float k = -rsqrtf(fmaxf(1.f - a.v * a.v, 1e-30f));
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] * k;
    return r;
}
__device__ __forceinline__ Dual dsin(const Dual& a) {
    Dual r;
    r.v = sinf(a.v);
    const float k = cosf(a.v);
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] * k;
    return r;
}
__device__ __forceinline__ Dual dcos(const Dual& a) {
    Dual r;
    r.v = cosf(a.v);
    const float k = -sinf(a.v);
#pragma unroll
    for (int i = 0; i < 9; ++i) r.d[i] = a.d[i] * k;
    return r;
}
// F.normalize(v, eps=1e-12): v / max(||v||, eps)
__device__ __forceinline__ void dnormalize3(Dual (&v)[3]) {
    Dual n = dsqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if (n.v < 1e-12f) n = dconst(1e-12f);
#pragma unroll
    for (int i = 0; i < 3; ++i) v[i] = v[i] / n;
}

// ------------------------------------------------------------------------------------------------
// PNP_NET pose-loss switches (gdrn_pose_switches).  Every loss is a per-crop partial in one of GDRN_POSE_SLOTS slots; the
// active slots, ascending, are the reference's loss_dict order (PyPMLoss entries, rot, centroid, z, trans, bind).
// ------------------------------------------------------------------------------------------------
enum PoseLoss { kLossL1 = 0, kLossSmoothL1 = 1, kLossMSE = 2, kLossL2 = 3 };
enum PmMode { kPmOff = -1, kPmR = 0, kPmRT = 1, kPmDisT = 2, kPmDisZ = 3, kPmDisTNoP = 4, kPmDisZNoP = 5 };
enum PoseSlot { kSlotPmR = 0, kSlotPmT = 1, kSlotPmZ = 2, kSlotNoP = 3, kSlotNoPZ = 4, kSlotRot = 5, kSlotCentroid = 6, kSlotZ = 7,
                kSlotTrans = 8, kSlotTransZ = 9, kSlotBind = 10 };

__host__ __device__ inline unsigned pose_slot_mask(const gdrn_pose_switches& sw) {
    unsigned m = (1u << kSlotCentroid) | (1u << kSlotZ);
    switch (sw.pm_mode) {
        case kPmR: case kPmRT: m |= 1u << kSlotPmR; break;
        case kPmDisT: m |= (1u << kSlotPmR) | (1u << kSlotPmT); break;
        case kPmDisZ: m |= (1u << kSlotPmR) | (1u << kSlotPmT) | (1u << kSlotPmZ); break;
        case kPmDisTNoP: m |= (1u << kSlotPmR) | (1u << kSlotNoP); break;
        case kPmDisZNoP: m |= (1u << kSlotPmR) | (1u << kSlotNoP) | (1u << kSlotNoPZ); break;
        default: break;
    }
    if (sw.rot_type >= 0) m |= 1u << kSlotRot;
    if (sw.trans_type >= 0) m |= sw.trans_disentangle ? (1u << kSlotTrans) | (1u << kSlotTransZ) : (1u << kSlotTrans);
    if (sw.bind_type >= 0) m |= 1u << kSlotBind;
    return m;
}

// loss_s = fac * sum_b part[b][s] / den.  Elementwise kinds take the mean over every element (the PM entries carry the
// reference's factor 3 over B n 3 elements: 1 / (B n)); L2 is the mean over B of per-crop norms (3 / B for the PM entries).
__host__ __device__ inline double pose_slot_den(const gdrn_pose_switches& sw, int s, int B, int n_pts, double* fac) {
    *fac = 1.0;
    const bool l2_pm = sw.pm_type == kLossL2;
    switch (s) {
        case kSlotPmR: case kSlotPmT: case kSlotPmZ:
            if (l2_pm) {
                *fac = 3.0;
                return (double)B;
            }
            return (double)B * n_pts;
        case kSlotNoP: return l2_pm ? (double)B : (sw.pm_mode == kPmDisTNoP ? 3.0 : 2.0) * B;
        case kSlotRot: return sw.rot_type == 1 ? 9.0 * B : (double)B;
        case kSlotCentroid: return sw.centroid_type == kLossL2 ? (double)B : 2.0 * B;
        case kSlotTrans:
            return sw.trans_type == kLossL2 ? (double)B : (sw.trans_disentangle ? 2.0 : 3.0) * B;
        case kSlotBind: return sw.bind_type == kLossL2 ? (double)B : 3.0 * B;
        default: return (double)B;  // z_noP, z, trans z: one element per crop
    }
}

// one residual e: value v and dv/de of L1 | Smooth-L1 (torch / fvcore: 0.5 e^2 / beta below beta, |e| - 0.5 beta above, L1 for
// beta < 1e-5) | MSE; for L2 v = e^2 and g = e (the norm and its 1 / ||e|| are applied per crop)
__device__ __forceinline__ void pose_elem(int kind, float e, float beta, float& v, float& g) {
    const float a = fabsf(e);
    const float sg = e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f);
    if (kind == kLossSmoothL1 && beta >= 1e-5f) {
        if (a < beta) {
            v = __fmul_rn(__fmul_rn(0.5f, a), a) / beta;
            g = e / beta;
        } else {
            v = a - __fmul_rn(0.5f, beta);
            g = sg;
        }
    } else if (kind == kLossMSE) {
        v = __fmul_rn(e, e);
        g = 2.f * e;
    } else if (kind == kLossL2) {
        v = __fmul_rn(e, e);
        g = e;
    } else {
        v = a;
        g = sg;
    }
}

// a group of n residuals of one loss entry of one crop: returns the crop's partial, d = coef * d(partial)/de.  L2: the norm
// sqrt(sum e^2) with d = coef e / ||e||, and d = 0 at ||e|| = 0 like torch.norm's gradient.
__device__ __forceinline__ float pose_group(int kind, float beta, const float* e, int n, float coef, float* d) {
    float s = 0.f;
    if (kind == kLossL2) {
        for (int i = 0; i < n; ++i) s += __fmul_rn(e[i], e[i]);
        const float nrm = sqrtf(s);
        const float c = nrm > 0.f ? coef / nrm : 0.f;
        for (int i = 0; i < n; ++i) d[i] = c * e[i];
        return nrm;
    }
    for (int i = 0; i < n; ++i) {
        float v, g;
        pose_elem(kind, e[i], beta, v, g);
        s += v;
        d[i] = coef * g;
    }
    return s;
}

struct PoseParams {
    const float* rot6d;   // [B][ld_pred] cols 0..5 (fc output fp32)
    const float* pred_t;  // [B][ld_pred] (pointer already offset to col 6)
    int ld_pred;
    const float* cams;      // [B][3][3]
    const float* centers;   // [B][2]
    const float* whs;       // [B][2]
    const float* ratios;    // [B]
    const float* extents;   // [B][3]
    const float* points;    // [B][n][3]
    const float* gt_rot;    // [B][3][3]
    const float* gt_trans;  // [B][3]
    const float* gt_ratio;  // [B][3]  (trans_ratio)
    const float* syms;      // device-resident symmetry table [rows][3][3] or null
    const int* sym_idx;     // [B][2] (first row, count) into syms, count 0 = no symmetry; null with syms
    const float* gw;        // [3]: upstream grads of loss_PM_R, loss_centroid, loss_z
    float* out_rot;         // [B][3][3]
    float* out_trans;       // [B][3]
    double* sums;           // [4]: PM abs sum, centroid abs sum, z abs sum, unused
    float* vis;             // [B][2]: re (deg), te per sample
    bf16* dy_hi;            // [B][64] gradient wrt the 9 FC outputs (rot6d | t), cols >= 9 zero
    bf16* dy_lo;
    int B, n_pts, do_loss;
    float eps;  // 1e-4 in the differentiable train decode (utils.py:208-236); 0 = exact normalisation of the test-time
                // decode (pose_from_pred_centroid_z.py:52-141 -> utils.py:39-94 axangle2mat)
    // EX only (gdrn_pose_loss_ex): the switches, per-crop partials [B][GDRN_POSE_SLOTS] instead of `sums`, and gw = the upstream
    // gradients of the active slots in slot order
    gdrn_pose_switches sw;
    float* part;
};

// The losses of gdrn_pose_loss_ex after the decode and the symmetric search (sRgt: the PM target, sRg0: the original R_gt that
// loss_rot and loss_bind use).  The per-point pass accumulates the three point-matching terms, dL/dR (G, as in the shipped
// kernel) and dL/dT (GT); L2 needs no second pass because its gradient is sum(e p^T) / ||e|| per crop.  Thread 0 then adds the
// per-crop losses on (R, T, pred_t) and contracts everything with the forward-mode Jacobians sJ (dR) and sJT (dT).
__device__ __forceinline__ void pose_loss_ex_tail(const PoseParams& p, const float* sR, const float* sRgt, const float* sRg0,
                                                  const float* sT, float (*sJ)[9], float (*sJT)[9], float* sG, float* sGT,
                                                  float* sAcc, float (*red)[4]) {
    const int b = blockIdx.x;
    const gdrn_pose_switches& sw = p.sw;
    const int mode = sw.pm_mode, kind = sw.pm_type;
    const float beta = sw.pm_beta;
    const float* Tgp = p.gt_trans + b * 3;
    const float Tp[3] = {sT[0], sT[1], sT[2]}, Tg[3] = {Tgp[0], Tgp[1], Tgp[2]};
    // weights * points (pm_loss.py:102-107): 1 / max extent, or exactly 1
    const float w = sw.pm_norm_extent ? 1.f / fmaxf(fmaxf(p.extents[b * 3], p.extents[b * 3 + 1]), p.extents[b * 3 + 2]) : 1.f;
    float acc[3] = {0.f, 0.f, 0.f}, G[9], GT[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 9; ++i) G[i] = 0.f;
    if (mode != kPmOff) {
        const float* pts = p.points + (long)b * p.n_pts * 3;
        for (int n = threadIdx.x; n < p.n_pts; n += blockDim.x) {
            const float px = pts[n * 3], py = pts[n * 3 + 1], pz = pts[n * 3 + 2];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float est = sR[i * 3] * px + sR[i * 3 + 1] * py + sR[i * 3 + 2] * pz;
                const float tgt = sRgt[i * 3] * px + sRgt[i * 3 + 1] * py + sRgt[i * 3 + 2] * pz;
                // rotation term: R p [+ t | + t_gt] against R_gt p [+ t_gt], each side weighted before the subtraction
                float e;
                if (mode == kPmRT) e = masked_diff(est + Tp[i], tgt + Tg[i], w);
                else if (mode == kPmDisT || mode == kPmDisZ) e = masked_diff(est + Tg[i], tgt + Tg[i], w);
                else e = masked_diff(est, tgt, w);
                float v, g;
                pose_elem(kind, e, beta, v, g);
                acc[0] += v;
                const float sg = g * w;
                G[i * 3] += sg * px;
                G[i * 3 + 1] += sg * py;
                G[i * 3 + 2] += sg * pz;
                if (mode == kPmRT) GT[i] += sg;
                // translation terms with points: R_gt p + t (DISENTANGLE_T), or with t_gt's z (xy) / x, y (z) for DISENTANGLE_Z,
                // whose other components are exactly 0 and are skipped
                if (mode == kPmDisT || mode == kPmDisZ) {
                    const float e1 = masked_diff(tgt + Tp[i], tgt + Tg[i], w);
                    pose_elem(kind, e1, beta, v, g);
                    acc[(mode == kPmDisZ && i == 2) ? 2 : 1] += v;
                    GT[i] += g * w;
                }
            }
        }
    }
    float vals[15];
#pragma unroll
    for (int j = 0; j < 3; ++j) vals[j] = acc[j];
#pragma unroll
    for (int j = 0; j < 9; ++j) vals[3 + j] = G[j];
#pragma unroll
    for (int j = 0; j < 3; ++j) vals[12 + j] = GT[j];
#pragma unroll
    for (int j = 0; j < 15; ++j) {
        float v = vals[j];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[j][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x < 15) {
        const float v = red[threadIdx.x][0] + red[threadIdx.x][1] + red[threadIdx.x][2] + red[threadIdx.x][3];
        if (threadIdx.x < 3) sAcc[threadIdx.x] = v;
        else if (threadIdx.x < 12) sG[threadIdx.x - 3] = v;
        else sGT[threadIdx.x - 12] = v;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;

    const unsigned mask = pose_slot_mask(sw);
    auto coef = [&](int s) {  // upstream gradient * fac / den of slot s
        double fac;
        const float den = (float)pose_slot_den(sw, s, p.B, p.n_pts, &fac);
        return p.gw[__popc(mask & ((1u << s) - 1u))] * (float)fac / den;
    };
    float* part = p.part + (long)b * GDRN_POSE_SLOTS;
    float g[16], GR[9], GTt[3] = {0.f, 0.f, 0.f}, d[3];
    for (int i = 0; i < 9; ++i) GR[i] = 0.f;
    for (int k = 0; k < 9; ++k) g[k] = 0.f;
    // ---- point matching (pm_loss.py:97-171)
    if (mode != kPmOff) {
        float c[3] = {0.f, 0.f, 0.f};
        for (int s = kSlotPmR; s <= kSlotPmZ; ++s) {
            if (!((mask >> s) & 1u)) continue;
            if (kind == kLossL2) {
                const float nrm = sqrtf(sAcc[s]);
                part[s] = nrm;
                c[s] = nrm > 0.f ? coef(s) / nrm : 0.f;
            } else {
                part[s] = sAcc[s];
                c[s] = coef(s);
            }
        }
        for (int k = 0; k < 9; ++k) {
            float s = 0.f;
            for (int ij = 0; ij < 9; ++ij) s += sG[ij] * sJ[ij][k];
            g[k] = c[0] * s;
        }
        if (mode == kPmRT)
            for (int i = 0; i < 3; ++i) GTt[i] += c[0] * sGT[i];
        if (mode == kPmDisT || mode == kPmDisZ)
            for (int i = 0; i < 3; ++i) GTt[i] += c[(mode == kPmDisZ && i == 2) ? 2 : 1] * sGT[i];
        // without points: loss_func(t, t_gt) on [B, 3], or on [B, 2] and [B] -- no weights, no factor 3, no PM_LW
        if (mode == kPmDisTNoP || mode == kPmDisZNoP) {
            const float e[3] = {Tp[0] - Tg[0], Tp[1] - Tg[1], Tp[2] - Tg[2]};
            if (mode == kPmDisTNoP) {
                part[kSlotNoP] = pose_group(kind, beta, e, 3, coef(kSlotNoP), d);
                for (int i = 0; i < 3; ++i) GTt[i] += d[i];
            } else {
                part[kSlotNoP] = pose_group(kind, beta, e, 2, coef(kSlotNoP), d);
                GTt[0] += d[0];
                GTt[1] += d[1];
                part[kSlotNoPZ] = pose_group(kind, beta, e + 2, 1, coef(kSlotNoPZ), d);
                GTt[2] += d[0];
            }
        }
    }
    // ---- loss_rot against the original R_gt (rot_loss.py:30-48): angular (1 - (tr(R R_gt^T) - 1) / 2) / 2, or mean (R - R_gt)^2
    if ((mask >> kSlotRot) & 1u) {
        const float c = coef(kSlotRot);
        if (sw.rot_type == 0) {
            float m[3];
            for (int i = 0; i < 3; ++i) m[i] = sR[i * 3] * sRg0[i * 3] + sR[i * 3 + 1] * sRg0[i * 3 + 1] + sR[i * 3 + 2] * sRg0[i * 3 + 2];
            const float cs = (m[0] + m[1] + m[2] - 1.f) / 2.f;
            part[kSlotRot] = (1.f - cs) / 2.f;
            for (int i = 0; i < 9; ++i) GR[i] += -0.25f * c * sRg0[i];
        } else {
            float s = 0.f;
            for (int i = 0; i < 9; ++i) {
                const float e = sR[i] - sRg0[i];
                s += __fmul_rn(e, e);
                GR[i] += 2.f * c * e;
            }
            part[kSlotRot] = s;
        }
    }
    // ---- centroid and z on the raw network output against trans_ratio (GDRN.py:439-471; L2 of the [B] z is its L1)
    const float* tp = p.pred_t + (long)b * p.ld_pred;
    const float* gr = p.gt_ratio + b * 3;
    const float ec[2] = {tp[0] - gr[0], tp[1] - gr[1]}, ez = tp[2] - gr[2];
    float dc[2], dz;
    part[kSlotCentroid] = pose_group(sw.centroid_type, 0.f, ec, 2, coef(kSlotCentroid), dc);
    part[kSlotZ] = pose_group(sw.z_type, 0.f, &ez, 1, coef(kSlotZ), &dz);
    // ---- translation (GDRN.py:474-500): xy and z, or all three (loss_trans_LPnP)
    if ((mask >> kSlotTrans) & 1u) {
        const float e[3] = {Tp[0] - Tg[0], Tp[1] - Tg[1], Tp[2] - Tg[2]};
        if (sw.trans_disentangle) {
            part[kSlotTrans] = pose_group(sw.trans_type, 0.f, e, 2, coef(kSlotTrans), d);
            GTt[0] += d[0];
            GTt[1] += d[1];
            part[kSlotTransZ] = pose_group(sw.trans_type, 0.f, e + 2, 1, coef(kSlotTransZ), d);
            GTt[2] += d[0];
        } else {
            part[kSlotTrans] = pose_group(sw.trans_type, 0.f, e, 3, coef(kSlotTrans), d);
            for (int i = 0; i < 3; ++i) GTt[i] += d[i];
        }
    }
    // ---- bind (GDRN.py:503-514): R^T t against R_gt^T t_gt (original R_gt)
    if ((mask >> kSlotBind) & 1u) {
        float e[3];
        for (int j = 0; j < 3; ++j) {
            const float pb = sR[j] * Tp[0] + sR[3 + j] * Tp[1] + sR[6 + j] * Tp[2];
            const float gb = sRg0[j] * Tg[0] + sRg0[3 + j] * Tg[1] + sRg0[6 + j] * Tg[2];
            e[j] = pb - gb;
        }
        part[kSlotBind] = pose_group(sw.bind_type, 0.f, e, 3, coef(kSlotBind), d);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                GR[i * 3 + j] += Tp[i] * d[j];
                GTt[i] += sR[i * 3 + j] * d[j];
            }
    }
    // ---- chain rule through the decode; the shipped configuration adds nothing here
    if ((mask & ~((1u << kSlotPmR) | (1u << kSlotCentroid) | (1u << kSlotZ))) != 0u || mode == kPmRT) {
        for (int k = 0; k < 9; ++k) {
            float s = 0.f;
            for (int ij = 0; ij < 9; ++ij) s += GR[ij] * sJ[ij][k];
            for (int i = 0; i < 3; ++i) s += GTt[i] * sJT[i][k];
            g[k] += s;
        }
    }
    g[6] += dc[0];
    g[7] += dc[1];
    g[8] += dz;
    for (int k = 9; k < 16; ++k) g[k] = 0.f;
    for (int k = 0; k < 64; k += 2) {
        const float a = k < 16 ? g[k] : 0.f, c = k + 1 < 16 ? g[k + 1] : 0.f;
        uint32_t h, l;
        split2(a, c, h, l);
        *reinterpret_cast<uint32_t*>(p.dy_hi + (long)b * 64 + k) = h;
        if (p.dy_lo != nullptr) *reinterpret_cast<uint32_t*>(p.dy_lo + (long)b * 64 + k) = l;
    }
}

// EX = false: the shipped configuration (r_only L1 PM normalised by extent, L1 centroid and z) with atomic fp64 sums;
// EX = true: every PNP_NET switch (gdrn_pose_switches), per-crop partials.  Both share the decode and the symmetric search.
template <bool EX>
__global__ void __launch_bounds__(128) pose_loss_kernel(const PoseParams p) {
    const int b = blockIdx.x;
    __shared__ float sR[9], sRgt[9], sG[9], sT[3];
    __shared__ float sJ[9][9];  // dR[i][j]/d input k
    __shared__ float red[EX ? 15 : 10][4];
    __shared__ float sJT[3][9], sRg0[9], sGT[3], sAcc[3];  // EX: dT[i]/d input k, the original (not symmetric) R_gt
    if (threadIdx.x == 0) {
        const float* r6 = p.rot6d + (long)b * p.ld_pred;
        const float* tp = p.pred_t + (long)b * p.ld_pred;
        Dual x[3], yr[3], z[3], y[3];
        for (int i = 0; i < 3; ++i) {
            x[i] = dvar(r6[i], i);
            yr[i] = dvar(r6[3 + i], 3 + i);
        }
        dnormalize3(x);
        z[0] = x[1] * yr[2] - x[2] * yr[1];
        z[1] = x[2] * yr[0] - x[0] * yr[2];
        z[2] = x[0] * yr[1] - x[1] * yr[0];
        dnormalize3(z);
        y[0] = z[1] * x[2] - z[2] * x[1];
        y[1] = z[2] * x[0] - z[0] * x[2];
        y[2] = z[0] * x[1] - z[1] * x[0];
        Dual Ra[3][3];
        for (int i = 0; i < 3; ++i) {
            Ra[i][0] = x[i];
            Ra[i][1] = y[i];
            Ra[i][2] = z[i];
        }
        // SITE translation
        const float* K = p.cams + b * 9;
        Dual t0 = dvar(tp[0], 6), t1 = dvar(tp[1], 7), t2 = dvar(tp[2], 8);
        Dual cx = t0 * p.whs[b * 2 + 0] + dconst(p.centers[b * 2 + 0]);
        Dual cy = t1 * p.whs[b * 2 + 1] + dconst(p.centers[b * 2 + 1]);
        Dual zz = t2 * p.ratios[b];
        Dual T[3];
        T[0] = zz * (cx - dconst(K[2])) / dconst(K[0]);
        T[1] = zz * (cy - dconst(K[5])) / dconst(K[4]);
        T[2] = zz;
        // allocentric -> egocentric
        Dual nT = dsqrt(T[0] * T[0] + T[1] * T[1] + T[2] * T[2]) + dconst(p.eps);
        Dual ray[3] = {T[0] / nT, T[1] / nT, T[2] / nT};
        Dual angle = dacos(ray[2]);
        Dual ax[3] = {-ray[1], ray[0], dconst(0.f)};
        Dual na = dsqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]) + dconst(p.eps);
        if (na.v <= 0.f) na = dconst(1.f);  // object exactly on the optical axis: angle = 0, rotation = identity (utils.py:62)
        for (int i = 0; i < 3; ++i) ax[i] = ax[i] / na;
        Dual half = angle * 0.5f;
        Dual sh = dsin(half);
        Dual q[4] = {dcos(half), ax[0] * sh, ax[1] * sh, ax[2] * sh};
        Dual nq = dsqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        for (int i = 0; i < 4; ++i) q[i] = q[i] / nq;
        Dual X = q[1] * 2.f, Y = q[2] * 2.f, Z = q[3] * 2.f;
        Dual wX = q[0] * X, wY = q[0] * Y, wZ = q[0] * Z;
        Dual xX = q[1] * X, xY = q[1] * Y, xZ = q[1] * Z;
        Dual yY = q[2] * Y, yZ = q[2] * Z, zZ = q[3] * Z;
        Dual one = dconst(1.f);
        Dual Rq[3][3] = {{one - (yY + zZ), xY - wZ, xZ + wY}, {xY + wZ, one - (xX + zZ), yZ - wX}, {xZ - wY, yZ + wX, one - (xX + yY)}};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                Dual e = Rq[i][0] * Ra[0][j] + Rq[i][1] * Ra[1][j] + Rq[i][2] * Ra[2][j];
                sR[i * 3 + j] = e.v;
                for (int k = 0; k < 9; ++k) sJ[i * 3 + j][k] = e.d[k];
                p.out_rot[b * 9 + i * 3 + j] = e.v;
            }
        for (int i = 0; i < 3; ++i) {
            sT[i] = T[i].v;
            p.out_trans[b * 3 + i] = T[i].v;
            if (EX)
                for (int k = 0; k < 9; ++k) sJT[i][k] = T[i].d[k];
        }
        if (p.do_loss) {
            // ground-truth rotation, optionally replaced by the closest symmetric equivalent (detached)
            float Rg[9];
            for (int i = 0; i < 9; ++i) Rg[i] = p.gt_rot[b * 9 + i];
            // logging: rotation error (deg) against the ORIGINAL gt, translation error
            {
                double tr = 0;
                for (int i = 0; i < 3; ++i)
                    for (int j = 0; j < 3; ++j) tr += (double)sR[i * 3 + j] * Rg[i * 3 + j];
                if (tr > 3) tr = 3;
                double c = 0.5 * (tr - 1.0);
                c = c > 1 ? 1 : (c < -1 ? -1 : c);
                p.vis[b * 2 + 0] = (float)(acos(c) * 57.29577951308232);
                double te = 0;
                for (int i = 0; i < 3; ++i) {
                    const double dd = (double)p.gt_trans[b * 3 + i] - sT[i];
                    te += dd * dd;
                }
                p.vis[b * 2 + 1] = (float)sqrt(te);
            }
            for (int i = 0; i < 9; ++i) sRgt[i] = Rg[i];
            if (EX)
                for (int i = 0; i < 9; ++i) sRg0[i] = Rg[i];
        }
    }
    __syncthreads();
    if (!p.do_loss) return;

    // closest symmetric ground truth (pose_utils.py:430-454: the FIRST candidate with the strictly smallest geodesic error,
    // the unmodified R_gt first), detached.  The K candidates (up to several hundred for discretised continuous
    // symmetries) are scanned by the whole CTA: trace(R^T R_gt S_k) = <M, S_k> with M = R_gt^T R, one acos per candidate,
    // then a lexicographic (error, index) minimum over the block.  The table `syms` is device-resident and shared by all
    // steps; `sym_idx[b] = (first row, count)` selects this crop's object (count 0 = asymmetric).
    if (p.syms != nullptr && p.sym_idx[2 * b + 1] > 0) {
        __shared__ double s_be[4];
        __shared__ int s_bk[4];
        const int k0 = p.sym_idx[2 * b], K = p.sym_idx[2 * b + 1];
        float M[9];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) M[i * 3 + j] = sRgt[0 * 3 + i] * sR[0 * 3 + j] + sRgt[1 * 3 + i] * sR[1 * 3 + j] + sRgt[2 * 3 + i] * sR[2 * 3 + j];
        double best;
        {
            double tr = (double)M[0] + (double)M[4] + (double)M[8];
            if (tr > 3) tr = 3;
            const double c = 0.5 * (tr - 1.0);
            best = acos(c > 1 ? 1 : (c < -1 ? -1 : c));
        }
        int bk = -1;
        for (int k = threadIdx.x; k < K; k += blockDim.x) {
            const float* S = p.syms + (long)(k0 + k) * 9;
            // the reference forms cand = R_gt S_k in fp32/fp64 and takes trace(R cand^T); <M, S_k> is the same sum re-associated
            double tr = 0;
#pragma unroll
            for (int i = 0; i < 9; ++i) tr += (double)M[i] * (double)__ldg(S + i);
            if (tr > 3) tr = 3;
            const double c = 0.5 * (tr - 1.0);
            const double e = acos(c > 1 ? 1 : (c < -1 ? -1 : c));
            if (e < best) {  // ascending k per thread: the first strict minimum is kept
                best = e;
                bk = k;
            }
        }
        // lexicographic min over (error, index); index -1 (the original R_gt) wins ties like the sequential scan
        for (int o = 16; o > 0; o >>= 1) {
            const double oe = __shfl_xor_sync(0xffffffffu, best, o);
            const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
            if (oe < best || (oe == best && ok < bk)) {
                best = oe;
                bk = ok;
            }
        }
        if ((threadIdx.x & 31) == 0) {
            s_be[threadIdx.x >> 5] = best;
            s_bk[threadIdx.x >> 5] = bk;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int wv = 1; wv < 4; ++wv)
                if (s_be[wv] < best || (s_be[wv] == best && s_bk[wv] < bk)) {
                    best = s_be[wv];
                    bk = s_bk[wv];
                }
            if (bk >= 0) {
                const float* S = p.syms + (long)(k0 + bk) * 9;
                float Rg[9], cand[9];
                for (int i = 0; i < 9; ++i) Rg[i] = sRgt[i];
                for (int i = 0; i < 3; ++i)
                    for (int j = 0; j < 3; ++j)
                        cand[i * 3 + j] = Rg[i * 3 + 0] * S[0 * 3 + j] + Rg[i * 3 + 1] * S[1 * 3 + j] + Rg[i * 3 + 2] * S[2 * 3 + j];
                for (int i = 0; i < 9; ++i) sRgt[i] = cand[i];
            }
        }
        __syncthreads();
    }

    if constexpr (EX) {
        pose_loss_ex_tail(p, sR, sRgt, sRg0, sT, sJ, sJT, sG, sGT, sAcc, red);
        return;
    }

    // point-matching loss (r_only, L1, normalised by max extent): sum |w (R p - Rgt p)|, and dL/dR = w sign(e) p^T
    const float w = 1.f / fmaxf(fmaxf(p.extents[b * 3], p.extents[b * 3 + 1]), p.extents[b * 3 + 2]);
    float acc = 0.f, G[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) G[i] = 0.f;
    float D[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) D[i] = sR[i] - sRgt[i];
    const float* pts = p.points + (long)b * p.n_pts * 3;
    for (int n = threadIdx.x; n < p.n_pts; n += blockDim.x) {
        const float px = pts[n * 3], py = pts[n * 3 + 1], pz = pts[n * 3 + 2];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            // reference computes est and tgt separately then subtracts; (R - Rgt) p is the same up to rounding
            const float est = sR[i * 3] * px + sR[i * 3 + 1] * py + sR[i * 3 + 2] * pz;
            const float tgt = sRgt[i * 3] * px + sRgt[i * 3 + 1] * py + sRgt[i * 3 + 2] * pz;
            const float e = masked_diff(est, tgt, w);
            acc += fabsf(e);
            const float sg = e > 0.f ? w : (e < 0.f ? -w : 0.f);
            G[i * 3] += sg * px;
            G[i * 3 + 1] += sg * py;
            G[i * 3 + 2] += sg * pz;
        }
    }
    (void)D;
    float vals[10];
    vals[0] = acc;
#pragma unroll
    for (int i = 0; i < 9; ++i) vals[1 + i] = G[i];
#pragma unroll
    for (int j = 0; j < 10; ++j) {
        float v = vals[j];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[j][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x < 9) sG[threadIdx.x] = red[1 + threadIdx.x][0] + red[1 + threadIdx.x][1] + red[1 + threadIdx.x][2] + red[1 + threadIdx.x][3];
    __syncthreads();
    if (threadIdx.x == 0) {
        const float pm = red[0][0] + red[0][1] + red[0][2] + red[0][3];
        const float* tp = p.pred_t + (long)b * p.ld_pred;
        const float* gr = p.gt_ratio + b * 3;
        const float e0 = tp[0] - gr[0], e1 = tp[1] - gr[1], e2 = tp[2] - gr[2];
        atomicAdd(p.sums + 0, (double)pm);
        atomicAdd(p.sums + 1, (double)(fabsf(e0) + fabsf(e1)));
        atomicAdd(p.sums + 2, (double)fabsf(e2));
        // gradients wrt (rot6d, t): loss_PM_R = 3 * sum / (B n 3); centroid = sum/(2B); z = sum/B
        const float cpm = p.gw[0] / ((float)p.B * (float)p.n_pts);
        float g[16];
        for (int k = 0; k < 9; ++k) {
            float s = 0.f;
            for (int ij = 0; ij < 9; ++ij) s += sG[ij] * sJ[ij][k];
            g[k] = cpm * s;
        }
        const float cc = p.gw[1] / (2.f * p.B), cz = p.gw[2] / (float)p.B;
        g[6] += cc * (e0 > 0.f ? 1.f : (e0 < 0.f ? -1.f : 0.f));
        g[7] += cc * (e1 > 0.f ? 1.f : (e1 < 0.f ? -1.f : 0.f));
        g[8] += cz * (e2 > 0.f ? 1.f : (e2 < 0.f ? -1.f : 0.f));
        for (int k = 9; k < 16; ++k) g[k] = 0.f;
        for (int k = 0; k < 64; k += 2) {
            const float a = k < 16 ? g[k] : 0.f, c = k + 1 < 16 ? g[k + 1] : 0.f;
            uint32_t h, l;
            split2(a, c, h, l);
            *reinterpret_cast<uint32_t*>(p.dy_hi + (long)b * 64 + k) = h;
            if (p.dy_lo != nullptr) *reinterpret_cast<uint32_t*>(p.dy_lo + (long)b * 64 + k) = l;
        }
    }
}

// losses[8] = coor_x, coor_y, coor_z, mask, region, PM_R, centroid, z ; vis_out[2] = mean re, mean te
// reg_slot: the pix_sums slot holding sum(region mask), 6, or 5 for the six-slot layout whose region mask is the xyz mask
__global__ void loss_finalize_kernel(const double* __restrict__ pix_sums, const double* __restrict__ pose_sums,
                                     const float* __restrict__ vis, float* __restrict__ losses, float* __restrict__ vis_out,
                                     int B, int HW, int n_pts, int reg_slot) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double fg = pix_sums[5] < 1.0 ? 1.0 : pix_sums[5];
    const double fg_reg = pix_sums[reg_slot] < 1.0 ? 1.0 : pix_sums[reg_slot];
    losses[0] = (float)(pix_sums[0] / fg);
    losses[1] = (float)(pix_sums[1] / fg);
    losses[2] = (float)(pix_sums[2] / fg);
    losses[3] = (float)(pix_sums[3] / ((double)B * HW));
    losses[4] = (float)(pix_sums[4] / fg_reg);
    losses[5] = (float)(pose_sums[0] / ((double)B * n_pts));
    losses[6] = (float)(pose_sums[1] / (2.0 * B));
    losses[7] = (float)(pose_sums[2] / (double)B);
    float re = 0.f, te = 0.f;
    for (int b = 0; b < B; ++b) {
        re += vis[b * 2];
        te += vis[b * 2 + 1];
    }
    vis_out[0] = re / B;
    vis_out[1] = te / B;
}

// losses[5 + n_pose]: the pixel losses as loss_finalize_kernel (region normaliser slot 6), then each active pose slot as the
// crop-ordered fp64 sum of its partials (no atomics: the same inputs give the same losses)
__global__ void loss_finalize_ex2_kernel(const double* __restrict__ pix_sums, const float* __restrict__ part,
                                         const float* __restrict__ vis, float* __restrict__ losses, float* __restrict__ vis_out,
                                         int B, int HW, int n_pts, const gdrn_pose_switches sw) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double fg = pix_sums[5] < 1.0 ? 1.0 : pix_sums[5];
    const double fg_reg = pix_sums[6] < 1.0 ? 1.0 : pix_sums[6];
    losses[0] = (float)(pix_sums[0] / fg);
    losses[1] = (float)(pix_sums[1] / fg);
    losses[2] = (float)(pix_sums[2] / fg);
    losses[3] = (float)(pix_sums[3] / ((double)B * HW));
    losses[4] = (float)(pix_sums[4] / fg_reg);
    const unsigned mask = pose_slot_mask(sw);
    int o = 5;
    for (int s = 0; s < GDRN_POSE_SLOTS; ++s) {
        if (!((mask >> s) & 1u)) continue;
        double sum = 0.0, fac;
        for (int b = 0; b < B; ++b) sum += (double)part[(long)b * GDRN_POSE_SLOTS + s];
        const double den = pose_slot_den(sw, s, B, n_pts, &fac);
        losses[o++] = (float)(fac == 1.0 ? sum / den : fac * sum / den);
    }
    float re = 0.f, te = 0.f;
    for (int b = 0; b < B; ++b) {
        re += vis[b * 2];
        te += vis[b * 2 + 1];
    }
    vis_out[0] = re / B;
    vis_out[1] = te / B;
}

}  // namespace gdrn

using namespace gdrn;

extern "C" int gdrn_head_glue_fwd_ex(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo,
                                     int B, int HW, int with_2d, int mask_out, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (with_2d && coord2d == nullptr) return set_error(GDRN_ERR_ARG, "head_glue_fwd: with_2d needs coord2d");
    if (mask_out != 1 && mask_out != 2) return set_error(GDRN_ERR_ARG, "head_glue_fwd: mask_out %d (1 or 2)", mask_out);
    const int grid = px_grid((long)B * HW);
#define GLUE(MO, W2D) head_glue_fwd_kernel<MO, W2D><<<grid, 128, 0, stream>>>(logits, coord2d, extents, (bf16*)out_hi, (bf16*)out_lo, B, HW)
    if (mask_out == 1) {
        if (with_2d) GLUE(1, true);
        else GLUE(1, false);
    } else {
        if (with_2d) GLUE(2, true);
        else GLUE(2, false);
    }
#undef GLUE
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_head_glue_fwd(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo,
                                  int B, int HW, int with_2d, void* stream_) {
    return gdrn_head_glue_fwd_ex(logits, coord2d, extents, out_hi, out_lo, B, HW, with_2d, 1, stream_);
}

extern "C" int gdrn_pnp_pack_input(const float* coor_feat, int c_feat, const float* region, int c_reg, const float* extents,
                                   void* out_hi, void* out_lo, int B, int HW, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (c_feat < 0 || c_reg < 0 || c_feat + c_reg > 72 || c_feat + c_reg < 1)
        return set_error(GDRN_ERR_ARG, "pnp_pack_input: %d + %d channels unsupported (1..72)", c_feat, c_reg);
    if (c_reg > 0 && region == nullptr) return set_error(GDRN_ERR_ARG, "pnp_pack_input: region missing");
    pnp_pack_input_kernel<<<px_grid((long)B * HW), 128, 0, stream>>>(coor_feat, c_feat, region, c_reg, extents, (bf16*)out_hi,
                                                                    (bf16*)out_lo, B, HW);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

// n_sums 7: the generalised layout; 6: the original one (slot 6 absent, region mask == xyz mask)
static int pixel_loss_launch(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_tgt, const float* m_reg,
                             const long long* labels, double* sums, int n_sums, int B, int HW, int mask_loss, cudaStream_t stream) {
    GDRN_CUDA_OK(cudaMemsetAsync(sums, 0, n_sums * sizeof(double), stream));
    const int grid = px_grid((long)B * HW);
    const bool sep = m_reg != m_xyz;
#define PIX(MODE, MO, SEP) \
    pixel_loss_fwd_kernel<MODE, MO, SEP><<<grid, 128, 0, stream>>>(logits, gt_xyz, m_xyz, m_tgt, m_reg, labels, sums, n_sums, B, HW)
    if (mask_loss == kMaskL1) {
        if (sep) PIX(kMaskL1, 1, true);
        else PIX(kMaskL1, 1, false);
    } else if (mask_loss == kMaskBCE) {
        if (sep) PIX(kMaskBCE, 1, true);
        else PIX(kMaskBCE, 1, false);
    } else {
        if (sep) PIX(kMaskCE, 2, true);
        else PIX(kMaskCE, 2, false);
    }
#undef PIX
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_pixel_loss_fwd_ex(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                                      const float* m_region, const long long* labels, double* sums, int B, int HW, int mask_loss,
                                      int mask_out, void* stream_) {
    if (int rc = check_mask_head("pixel_loss_fwd", mask_loss, mask_out)) return rc;
    return pixel_loss_launch(logits, gt_xyz, m_xyz, m_mask, m_region, labels, sums, 7, B, HW, mask_loss,
                             reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gdrn_pixel_loss_fwd(const float* logits, const float* gt_xyz, const float* m_visib, const float* m_trunc,
                                   const long long* labels, double* sums, int B, int HW, void* stream_) {
    return pixel_loss_launch(logits, gt_xyz, m_visib, m_trunc, m_visib, labels, sums, 6, B, HW, kMaskL1,
                             reinterpret_cast<cudaStream_t>(stream_));
}

template <int MODE, int MO, bool SEP>
static void head_bwd_launch(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_tgt, const float* m_reg,
                            const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                            const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, cudaStream_t stream) {
    const int grid = px_grid((long)B * HW);
    if (with_2d)
        head_bwd_kernel<MODE, MO, SEP, true><<<grid, 128, 0, stream>>>(logits, gt_xyz, m_xyz, m_tgt, m_reg, labels, sums, gw,
                                                                       (const bf16*)din_hi, (const bf16*)din_lo, extents,
                                                                       (bf16*)out_hi, (bf16*)out_lo, B, HW);
    else
        head_bwd_kernel<MODE, MO, SEP, false><<<grid, 128, 0, stream>>>(logits, gt_xyz, m_xyz, m_tgt, m_reg, labels, sums, gw,
                                                                        (const bf16*)din_hi, (const bf16*)din_lo, extents,
                                                                        (bf16*)out_hi, (bf16*)out_lo, B, HW);
}

extern "C" int gdrn_head_bwd_ex(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                                const float* m_region, const long long* labels, const double* sums, const float* gw,
                                const void* din_hi, const void* din_lo, const float* extents, void* out_hi, void* out_lo, int B,
                                int HW, int with_2d, int mask_loss, int mask_out, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (int rc = check_mask_head("head_bwd", mask_loss, mask_out)) return rc;
    const bool sep = m_region != m_xyz;
#define HB(MODE, MO, SEP) \
    head_bwd_launch<MODE, MO, SEP>(logits, gt_xyz, m_xyz, m_mask, m_region, labels, sums, gw, din_hi, din_lo, extents, out_hi, out_lo, B, HW, with_2d, stream)
    if (mask_loss == kMaskL1) {
        if (sep) HB(kMaskL1, 1, true);
        else HB(kMaskL1, 1, false);
    } else if (mask_loss == kMaskBCE) {
        if (sep) HB(kMaskBCE, 1, true);
        else HB(kMaskBCE, 1, false);
    } else {
        if (sep) HB(kMaskCE, 2, true);
        else HB(kMaskCE, 2, false);
    }
#undef HB
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_head_bwd(const float* logits, const float* gt_xyz, const float* m_visib, const float* m_trunc,
                             const long long* labels, const double* sums, const float* gw, const void* din_hi,
                             const void* din_lo, const float* extents, void* out_hi, void* out_lo, int B, int HW,
                             int with_2d, void* stream_) {
    // the same mask pointer for xyz and region: the kernel reads only sums[5], so six-slot buffers stay valid
    return gdrn_head_bwd_ex(logits, gt_xyz, m_visib, m_trunc, m_visib, labels, sums, gw, din_hi, din_lo, extents, out_hi, out_lo, B,
                            HW, with_2d, kMaskL1, 1, stream_);
}

extern "C" int gdrn_head_glue_fwd_ex2(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo,
                                      int B, int HW, int with_2d, int mask_out, int num_regions, int region_att, int pnp_ld,
                                      void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (int rc = check_regions("head_glue_fwd", num_regions, region_att, pnp_ld)) return rc;
    if (int rc = check_pnp_ld("head_glue_fwd", with_2d, num_regions, region_att, pnp_ld)) return rc;
    if (with_2d && coord2d == nullptr) return set_error(GDRN_ERR_ARG, "head_glue_fwd: with_2d needs coord2d");
    if (mask_out != 1 && mask_out != 2) return set_error(GDRN_ERR_ARG, "head_glue_fwd: mask_out %d (1 or 2)", mask_out);
    const int grid = px_grid((long)B * HW);
#define GLUE(MO, W2D, ATT)                                                                                                     \
    head_glue_fwd2_kernel<MO, W2D, ATT><<<grid, 128, 0, stream>>>(logits, coord2d, extents, (bf16*)out_hi, (bf16*)out_lo, B, HW, \
                                                                  num_regions, pnp_ld)
#define GLUE_A(MO, W2D) \
    if (region_att) GLUE(MO, W2D, true); \
    else GLUE(MO, W2D, false)
    if (mask_out == 1) {
        if (with_2d) GLUE_A(1, true);
        else GLUE_A(1, false);
    } else {
        if (with_2d) GLUE_A(2, true);
        else GLUE_A(2, false);
    }
#undef GLUE_A
#undef GLUE
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_pnp_pack_input_ex(const float* coor_feat, int c_feat, const float* region, int c_reg, const float* extents,
                                      void* out_hi, void* out_lo, int B, int HW, int pnp_ld, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (c_feat < 0 || c_reg < 0 || c_feat + c_reg > 72 || c_feat + c_reg < 1)
        return set_error(GDRN_ERR_ARG, "pnp_pack_input: %d + %d channels unsupported (1..72)", c_feat, c_reg);
    if (pnp_ld != (c_feat + c_reg + 63) / 64 * 64)
        return set_error(GDRN_ERR_ARG, "pnp_pack_input: pnp_ld %d for %d channels (want %d)", pnp_ld, c_feat + c_reg,
                         (c_feat + c_reg + 63) / 64 * 64);
    if (c_reg > 0 && region == nullptr) return set_error(GDRN_ERR_ARG, "pnp_pack_input: region missing");
    pnp_pack_input2_kernel<false><<<px_grid((long)B * HW), 128, 0, stream>>>(coor_feat, c_feat, region, c_reg, extents, (bf16*)out_hi,
                                                                      (bf16*)out_lo, B, HW, pnp_ld);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_pixel_loss_fwd_ex2(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                                       const float* m_region, const long long* labels, double* sums, int B, int HW, int mask_loss,
                                       int mask_out, int num_regions, int region_att, int pnp_ld, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (int rc = check_mask_head("pixel_loss_fwd", mask_loss, mask_out)) return rc;
    if (int rc = check_regions("pixel_loss_fwd", num_regions, region_att, pnp_ld)) return rc;
    GDRN_CUDA_OK(cudaMemsetAsync(sums, 0, 7 * sizeof(double), stream));
    const int grid = px_grid((long)B * HW);
    const bool sep = m_region != m_xyz;
#define PIX(MODE, MO, SEP) \
    pixel_loss_fwd2_kernel<MODE, MO, SEP><<<grid, 128, 0, stream>>>(logits, gt_xyz, m_xyz, m_mask, m_region, labels, sums, B, HW, num_regions)
    if (mask_loss == kMaskL1) {
        if (sep) PIX(kMaskL1, 1, true);
        else PIX(kMaskL1, 1, false);
    } else if (mask_loss == kMaskBCE) {
        if (sep) PIX(kMaskBCE, 1, true);
        else PIX(kMaskBCE, 1, false);
    } else {
        if (sep) PIX(kMaskCE, 2, true);
        else PIX(kMaskCE, 2, false);
    }
#undef PIX
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

template <int MODE, int MO, bool SEP>
static void head_bwd2_launch(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_tgt, const float* m_reg,
                             const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                             const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, int nreg, int att,
                             int pnp_ld, cudaStream_t stream) {
    const int grid = px_grid((long)B * HW);
#define HB2(W2D, ATT)                                                                                                              \
    head_bwd2_kernel<MODE, MO, SEP, W2D, ATT><<<grid, 128, 0, stream>>>(logits, gt_xyz, m_xyz, m_tgt, m_reg, labels, sums, gw,      \
                                                                        (const bf16*)din_hi, (const bf16*)din_lo, extents,          \
                                                                        (bf16*)out_hi, (bf16*)out_lo, B, HW, nreg, pnp_ld)
    if (with_2d) {
        if (att) HB2(true, true);
        else HB2(true, false);
    } else {
        if (att) HB2(false, true);
        else HB2(false, false);
    }
#undef HB2
}

extern "C" int gdrn_head_bwd_ex2(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                                 const float* m_region, const long long* labels, const double* sums, const float* gw,
                                 const void* din_hi, const void* din_lo, const float* extents, void* out_hi, void* out_lo, int B,
                                 int HW, int with_2d, int mask_loss, int mask_out, int num_regions, int region_att, int pnp_ld,
                                 void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (int rc = check_mask_head("head_bwd", mask_loss, mask_out)) return rc;
    if (int rc = check_regions("head_bwd", num_regions, region_att, pnp_ld)) return rc;
    if (int rc = check_pnp_ld("head_bwd", with_2d, num_regions, region_att, pnp_ld)) return rc;
    const bool sep = m_region != m_xyz;
    if (num_regions == kNumReg && region_att)  // the shipped head: the kernels of gdrn_head_bwd_ex, bit for bit
        return gdrn_head_bwd_ex(logits, gt_xyz, m_xyz, m_mask, m_region, labels, sums, gw, din_hi, din_lo, extents, out_hi, out_lo,
                                B, HW, with_2d, mask_loss, mask_out, stream_);
#define HB(MODE, MO, SEP)                                                                                                  \
    head_bwd2_launch<MODE, MO, SEP>(logits, gt_xyz, m_xyz, m_mask, m_region, labels, sums, gw, din_hi, din_lo, extents, out_hi, \
                                    out_lo, B, HW, with_2d, num_regions, region_att, pnp_ld, stream)
    if (mask_loss == kMaskL1) {
        if (sep) HB(kMaskL1, 1, true);
        else HB(kMaskL1, 1, false);
    } else if (mask_loss == kMaskBCE) {
        if (sep) HB(kMaskBCE, 1, true);
        else HB(kMaskBCE, 1, false);
    } else {
        if (sep) HB(kMaskCE, 2, true);
        else HB(kMaskCE, 2, false);
    }
#undef HB
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_pose_loss(const float* pred, int ld_pred, const float* cams, const float* centers, const float* whs,
                              const float* ratios, const float* extents, const float* points, const float* gt_rot,
                              const float* gt_trans, const float* gt_ratio, const float* syms, const int* sym_idx,
                              const float* gw, float* out_rot, float* out_trans, double* sums, float* vis, void* dy_hi,
                              void* dy_lo, int B, int n_pts, int do_loss, float eps, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    PoseParams p;
    p.rot6d = pred;
    p.pred_t = pred + 6;
    p.ld_pred = ld_pred;
    p.cams = cams;
    p.centers = centers;
    p.whs = whs;
    p.ratios = ratios;
    p.extents = extents;
    p.points = points;
    p.gt_rot = gt_rot;
    p.gt_trans = gt_trans;
    p.gt_ratio = gt_ratio;
    p.syms = syms;
    p.sym_idx = sym_idx;
    p.gw = gw;
    p.out_rot = out_rot;
    p.out_trans = out_trans;
    p.sums = sums;
    p.vis = vis;
    p.dy_hi = (bf16*)dy_hi;
    p.dy_lo = (bf16*)dy_lo;
    p.B = B;
    p.n_pts = n_pts;
    p.do_loss = do_loss;
    p.eps = eps;
    if (do_loss) GDRN_CUDA_OK(cudaMemsetAsync(sums, 0, 4 * sizeof(double), stream));
    pose_loss_kernel<false><<<B, 128, 0, stream>>>(p);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

static int check_pose_switches(const char* fn, const gdrn_pose_switches& sw) {
    const auto kind3 = [](int t) { return t == kLossL1 || t == kLossMSE || t == kLossL2; };  // L1 | MSE | L2
    if (sw.pm_mode < kPmOff || sw.pm_mode > kPmDisZNoP) return set_error(GDRN_ERR_ARG, "%s: pm_mode %d", fn, sw.pm_mode);
    if (sw.pm_type < kLossL1 || sw.pm_type > kLossL2) return set_error(GDRN_ERR_ARG, "%s: pm_type %d", fn, sw.pm_type);
    if (sw.rot_type < -1 || sw.rot_type > 1) return set_error(GDRN_ERR_ARG, "%s: rot_type %d", fn, sw.rot_type);
    if (!kind3(sw.centroid_type) || !kind3(sw.z_type)) return set_error(GDRN_ERR_ARG, "%s: centroid / z loss type", fn);
    if ((sw.trans_type != -1 && !kind3(sw.trans_type)) || (sw.bind_type != -1 && !kind3(sw.bind_type)))
        return set_error(GDRN_ERR_ARG, "%s: trans / bind loss type", fn);
    return 0;
}

extern "C" int gdrn_pose_loss_count(gdrn_pose_switches sw) { return __builtin_popcount(pose_slot_mask(sw)); }

extern "C" int gdrn_pose_loss_ex(const float* pred, int ld_pred, const float* cams, const float* centers, const float* whs,
                                 const float* ratios, const float* extents, const float* points, const float* gt_rot,
                                 const float* gt_trans, const float* gt_ratio, const float* syms, const int* sym_idx,
                                 const float* gw, float* out_rot, float* out_trans, float* part, float* vis, void* dy_hi,
                                 void* dy_lo, int B, int n_pts, gdrn_pose_switches sw, void* stream_) {
    if (int rc = check_pose_switches("pose_loss_ex", sw)) return rc;
    if (part == nullptr || gw == nullptr || points == nullptr) return set_error(GDRN_ERR_ARG, "pose_loss_ex: part, gw and points are required");
    PoseParams p;
    p.rot6d = pred;
    p.pred_t = pred + 6;
    p.ld_pred = ld_pred;
    p.cams = cams;
    p.centers = centers;
    p.whs = whs;
    p.ratios = ratios;
    p.extents = extents;
    p.points = points;
    p.gt_rot = gt_rot;
    p.gt_trans = gt_trans;
    p.gt_ratio = gt_ratio;
    p.syms = syms;
    p.sym_idx = sym_idx;
    p.gw = gw;
    p.out_rot = out_rot;
    p.out_trans = out_trans;
    p.sums = nullptr;
    p.vis = vis;
    p.dy_hi = (bf16*)dy_hi;
    p.dy_lo = (bf16*)dy_lo;
    p.B = B;
    p.n_pts = n_pts;
    p.do_loss = 1;
    p.eps = 1e-4f;
    p.sw = sw;
    p.part = part;
    pose_loss_kernel<true><<<B, 128, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_loss_finalize_ex2(const double* pix_sums, const float* part, const float* vis, float* losses, float* vis_out,
                                      int B, int HW, int n_pts, gdrn_pose_switches sw, void* stream_) {
    if (int rc = check_pose_switches("loss_finalize_ex2", sw)) return rc;
    loss_finalize_ex2_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(pix_sums, part, vis, losses, vis_out, B, HW,
                                                                                     n_pts, sw);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

static int loss_finalize_launch(const double* pix_sums, const double* pose_sums, const float* vis, float* losses, float* vis_out,
                                int B, int HW, int n_pts, int reg_slot, cudaStream_t stream) {
    loss_finalize_kernel<<<1, 32, 0, stream>>>(pix_sums, pose_sums, vis, losses, vis_out, B, HW, n_pts, reg_slot);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_loss_finalize_ex(const double* pix_sums, const double* pose_sums, const float* vis, float* losses,
                                     float* vis_out, int B, int HW, int n_pts, void* stream_) {
    return loss_finalize_launch(pix_sums, pose_sums, vis, losses, vis_out, B, HW, n_pts, 6, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gdrn_loss_finalize(const double* pix_sums, const double* pose_sums, const float* vis, float* losses,
                                  float* vis_out, int B, int HW, int n_pts, void* stream_) {
    return loss_finalize_launch(pix_sums, pose_sums, vis, losses, vis_out, B, HW, n_pts, 5, reinterpret_cast<cudaStream_t>(stream_));
}
