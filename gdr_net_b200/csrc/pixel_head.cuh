// Per-pixel head kernels shared by losses.cu (the plain _ex2 entry points) and dropblock.cu (the same kernels with DropBlock
// on the Patch-PnP input): the logit-row helpers, the glue, the stand-alone Patch-PnP input packing and the fused head
// backward for any region count, and the argument checks of their entry points.
#pragma once
#include <math.h>

#include "../../include/gdrn_b200.h"
#include "gdrn_internal.h"
#include "ptx.cuh"

namespace gdrn {

typedef __nv_bfloat16 bf16;
constexpr int kLogitLd = 72;   // 68 + MO logits padded to 72 floats per pixel
constexpr int kPnpLd = 128;    // Patch-PnP input channels padded to 128
constexpr int kNumReg = 64;    // foreground regions (region logits: bg + 64)

// Mask head (ROT_HEAD.MASK_LOSS_TYPE, GDRN.py:376-385): MO = 1 mask logit for L1 and BCE, MO = 2 for CE.  A logit row is
// mask [0, MO) | xyz [MO, MO + 3) | bg MO + 3 | regions [MO + 4, MO + 68)  (cdpn_rot_head_region.py:185-192).
enum MaskLoss { kMaskL1 = 0, kMaskBCE = 1, kMaskCE = 2 };

// Per-pixel mask loss against the target t (GT mask value): |z - t|; BCEWithLogits in the stable form
// max(z, 0) - z t + log1p(exp(-|z|)); CrossEntropy over (z0, z1) with label (int) t, the reference's .long() truncation.
template <int MODE>
__device__ __forceinline__ float mask_loss(const float (&z)[kLogitLd], float t) {
    if (MODE == kMaskL1) return fabsf(z[0] - t);
    if (MODE == kMaskBCE) return fmaxf(z[0], 0.f) - z[0] * t + log1pf(expf(-fabsf(z[0])));
    const float lse = fmaxf(z[0], z[1]) + log1pf(expf(-fabsf(z[0] - z[1])));
    return lse - ((int)t == 1 ? z[1] : z[0]);
}

// logistic sigmoid without overflow: exp of a non-positive argument only
__device__ __forceinline__ float sigmoid_stable(float x) {
    const float e = expf(-fabsf(x));
    return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}

// d(mask loss)/d(mask logits) scaled by c = upstream gradient / (B HW): sign(z - t); sigmoid(z) - t; softmax - onehot
template <int MODE>
__device__ __forceinline__ void mask_loss_bwd(const float (&z)[kLogitLd], float t, float c, float (&d)[72]) {
    if (MODE == kMaskL1) {
        const float e = z[0] - t;
        d[0] = c * (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f));
    } else if (MODE == kMaskBCE) {
        d[0] = c * (sigmoid_stable(z[0]) - t);
    } else {
        const int lab = (int)t;
        d[0] = c * (sigmoid_stable(z[0] - z[1]) - (lab == 1 ? 0.f : 1.f));
        d[1] = c * (sigmoid_stable(z[1] - z[0]) - (lab == 1 ? 1.f : 0.f));
    }
}

__device__ __forceinline__ void store_row_bf16(bf16* hi, bf16* lo, long row, int ld, const float* v, int n) {
    // n multiple of 8, v[n] in registers/local
    for (int j = 0; j < n; j += 8) {
        uint32_t h[4], l[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            split2(v[j + 2 * q], v[j + 2 * q + 1], h[q], l[q]);
        }
        *reinterpret_cast<uint4*>(hi + row * ld + j) = make_uint4(h[0], h[1], h[2], h[3]);
        if (lo != nullptr) *reinterpret_cast<uint4*>(lo + row * ld + j) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

__device__ __forceinline__ void load_logits(const float* __restrict__ logits, long pix, float (&z)[kLogitLd]) {
    const float4* src = reinterpret_cast<const float4*>(logits + pix * kLogitLd);
#pragma unroll
    for (int j = 0; j < kLogitLd / 4; ++j) {
        const float4 q = __ldg(src + j);
        z[4 * j] = q.x;
        z[4 * j + 1] = q.y;
        z[4 * j + 2] = q.z;
        z[4 * j + 3] = q.w;
    }
}

// a * w - b * w with both products rounded, like the reference's l1_loss(a * w, b * w): exactly 0 when a == b, so the L1
// gradient sign(0) = 0 there.  Without __fmul_rn the compiler contracts it to fma(a, w, -(b * w)), which leaves the rounding
// error of b * w and turns that 0 into a +-1 of arbitrary sign.
__device__ __forceinline__ float masked_diff(float a, float b, float w) { return __fmul_rn(a, w) - __fmul_rn(b, w); }

// ------------------------------------------------------------------------------------------------
// Any region count R = ROT_HEAD.NUM_REGIONS in 2..64, with or without region attention (PNP_NET.REGION_ATTENTION).
// A logit row is mask [0, MO) | xyz [MO, MO + 3) | bg MO + 3 | R regions [MO + 4, MO + 4 + R): N = MO + 4 + R <= 70 of the 72
// floats are written by the output conv, the rest of the row is never initialised.  The 65-slot loops below stay fully
// unrolled over compile-time indices (no local memory) and drop slot k > R with a select, never with a 0 weight: the unwritten
// columns may hold NaN, and NaN * 0 = NaN.  The Patch-PnP input is xyz | coord2d (W2D) | softmax_R (ATT), nIn channels in
// rows of pnp_ld = round_up(nIn, 64) = 64 or 128 16-bit values, the padding zero.
//
// Stores the first 64 values of v and, for a 128-wide row, v[64..71] and zeros in 72..127.
__device__ __forceinline__ void store_pnp_row(bf16* hi, bf16* lo, long row, int ld, const float (&v)[72]) {
    store_row_bf16(hi, lo, row, ld, v, 64);
    if (ld == 128) {
        store_row_bf16(hi + 64, lo != nullptr ? lo + 64 : nullptr, row, ld, v + 64, 8);
        const uint4 zz = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 72; j < 128; j += 8) {
            *reinterpret_cast<uint4*>(hi + row * ld + j) = zz;
            if (lo != nullptr) *reinterpret_cast<uint4*>(lo + row * ld + j) = zz;
        }
    }
}

// the first n floats of a logit row (n a multiple of 4, compile-time)
template <int N>
__device__ __forceinline__ void load_logits_head(const float* __restrict__ logits, long pix, float (&z)[kLogitLd]) {
    const float4* src = reinterpret_cast<const float4*>(logits + pix * kLogitLd);
#pragma unroll
    for (int j = 0; j < N / 4; ++j) {
        const float4 q = __ldg(src + j);
        z[4 * j] = q.x;
        z[4 * j + 1] = q.y;
        z[4 * j + 2] = q.z;
        z[4 * j + 3] = q.w;
    }
}

// channels [0, n) of a Patch-PnP input gradient row (hi + lo planes), n a multiple of 8 up to 72 (compile-time after inlining).
// A 64-wide row has no channels 64..71: that chunk re-reads 56..63, which can only feed region slots k >= nreg (nIn <= 64),
// and the callers drop those with selects.
__device__ __forceinline__ void load_din(const bf16* __restrict__ din_hi, const bf16* __restrict__ din_lo, long pix, int ld,
                                         float (&g)[72], int n) {
#pragma unroll
    for (int j = 0; j < n; j += 8) {
        const int col = (j < 64 || ld == 128) ? j : 56;
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(din_hi + pix * ld + col));
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) unpack_hi2(w[t], g[j + 2 * t], g[j + 2 * t + 1]);
        if (din_lo != nullptr) {
            const uint4 q2 = __ldg(reinterpret_cast<const uint4*>(din_lo + pix * ld + col));
            const uint32_t w2[4] = {q2.x, q2.y, q2.z, q2.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                float ra, rb;
                unpack_lo2(w2[t], ra, rb);
                g[j + 2 * t] += ra;
                g[j + 2 * t + 1] += rb;
            }
        }
    }
}

// DB: DropBlock on the Patch-PnP input (conv_pnp_net.py:128-142, dropblock.py): every valid channel of pixel pix is multiplied
// by keep[pix] * scale[0] in fp32 (gdrn_dropblock_step), the padding channels stay 0.
template <int MO, bool W2D, bool ATT, bool DB = false>
__global__ void __launch_bounds__(128) head_glue_fwd2_kernel(const float* __restrict__ logits, const float* __restrict__ coord2d,
                                                             const float* __restrict__ extents, bf16* __restrict__ out_hi,
                                                             bf16* __restrict__ out_lo, int B, int HW, int nreg, int pnp_ld,
                                                             const uint8_t* __restrict__ keep = nullptr,
                                                             const float* __restrict__ scale = nullptr) {
    const long total = (long)B * HW;
    const float db_scale = DB ? __ldg(scale) : 1.f;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < total; pix += (long)gridDim.x * blockDim.x) {
        const int b = (int)(pix / HW);
        const int hw = (int)(pix - (long)b * HW);
        float z[kLogitLd];
        if (ATT) load_logits(logits, pix, z);
        else load_logits_head<8>(logits, pix, z);  // mask and xyz only
        float o[72];
#pragma unroll
        for (int j = 0; j < 72; ++j) o[j] = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j) o[j] = (z[MO + j] - 0.5f) * __ldg(extents + b * 3 + j);
        constexpr int RO = W2D ? 5 : 3;  // first region channel
        if (W2D) {
            o[3] = __ldg(coord2d + ((long)b * 2 + 0) * HW + hw);
            o[4] = __ldg(coord2d + ((long)b * 2 + 1) * HW + hw);
        }
        if (ATT) {
            float m = -INFINITY;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) m = k < nreg ? fmaxf(m, z[MO + 4 + k]) : m;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) {
                o[RO + k] = k < nreg ? expf(z[MO + 4 + k] - m) : 0.f;
                s += o[RO + k];
            }
            const float inv = 1.f / s;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) o[RO + k] *= inv;
        }
        if (DB) {
            const float f = (float)__ldg(keep + pix) * db_scale;
            const int nin = RO + (ATT ? nreg : 0);
#pragma unroll
            for (int j = 0; j < 72; ++j) o[j] = j < nin ? o[j] * f : o[j];
        }
        store_pnp_row(out_hi, out_lo, pix, pnp_ld, o);
    }
}

// Patch-PnP input packing for the stand-alone ConvPnPNet.forward into rows of pnp_ld (64 or 128) channels; otherwise
// pnp_pack_input_kernel.  DB as head_glue_fwd2_kernel.
template <bool DB = false>
__global__ void __launch_bounds__(128) pnp_pack_input2_kernel(const float* __restrict__ coor, int c_feat,
                                                              const float* __restrict__ region, int c_reg,
                                                              const float* __restrict__ extents, bf16* __restrict__ out_hi,
                                                              bf16* __restrict__ out_lo, int B, int HW, int pnp_ld,
                                                              const uint8_t* __restrict__ keep = nullptr,
                                                              const float* __restrict__ scale = nullptr) {
    const long total = (long)B * HW;
    const float db_scale = DB ? __ldg(scale) : 1.f;
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
        if (DB) {
            const float f = (float)__ldg(keep + pix) * db_scale;
#pragma unroll
            for (int k = 0; k < 72; ++k) o[k] = k < c_feat + c_reg ? o[k] * f : o[k];
        }
        store_pnp_row(out_hi, out_lo, pix, pnp_ld, o);
    }
}

// head_bwd_kernel for nreg regions: d_logits [P][128] (columns >= MO + 4 + nreg zero) from the pixel losses and, with ATT, the
// softmax_R backward of the Patch-PnP input gradient din [P][pnp_ld]; without ATT only din's xyz (+ coord2d) channels are read.
// DB: din is the gradient of the DropBlock output; every row read is multiplied by keep[pix] * scale[0] first.
template <int MODE, int MO, bool SEP, bool W2D, bool ATT, bool DB = false>
__global__ void __launch_bounds__(128) head_bwd2_kernel(const float* __restrict__ logits, const float* __restrict__ gt_xyz,
                                                        const float* __restrict__ m_xyz, const float* __restrict__ m_tgt,
                                                        const float* __restrict__ m_reg, const long long* __restrict__ labels,
                                                        const double* __restrict__ sums,
                                                        const float* __restrict__ gw, const bf16* __restrict__ din_hi,
                                                        const bf16* __restrict__ din_lo, const float* __restrict__ extents,
                                                        bf16* __restrict__ out_hi, bf16* __restrict__ out_lo, int B, int HW, int nreg,
                                                        int pnp_ld, const uint8_t* __restrict__ keep = nullptr,
                                                        const float* __restrict__ scale = nullptr) {
    const long total = (long)B * HW;
    const float db_scale = DB ? __ldg(scale) : 1.f;
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
        mask_loss_bwd<MODE>(z, mt, gwm * inv_all, d);
        // the xyz (+ coord2d) channels of din; with attention the region channels follow after the region CE
        float gin[72];
        if (din_hi != nullptr) {
            load_din(din_hi, din_lo, pix, pnp_ld, gin, 8);
            if (DB) {
                const float f = (float)__ldg(keep + pix) * db_scale;
#pragma unroll
                for (int j = 0; j < 8; ++j) gin[j] *= f;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) gin[j] = 0.f;
        }
        const float gws[3] = {gwx, gwy, gwz};
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float e = masked_diff(z[MO + j], __ldg(gt_xyz + ((long)b * 3 + j) * HW + hw), mv);
            const float sg = e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f);
            d[MO + j] = gws[j] * inv_fg * sg * mv + gin[j] * __ldg(extents + b * 3 + j);
        }
        // region CE over nreg + 1 (masked logits); slots k > nreg get 0
        {
            float mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < 65; ++k) mx = k <= nreg ? fmaxf(mx, z[MO + 3 + k] * mr) : mx;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 65; ++k) {
                d[MO + 3 + k] = k <= nreg ? expf(z[MO + 3 + k] * mr - mx) : 0.f;
                s += d[MO + 3 + k];
            }
            const float c = gwr * inv_reg * mr;
            const float inv = 1.f / s;
            const int lab = (int)(__ldg(labels + pix) * (long long)mr);
#pragma unroll
            for (int k = 0; k < 65; ++k) d[MO + 3 + k] = k <= nreg ? c * (d[MO + 3 + k] * inv - (k == lab ? 1.f : 0.f)) : 0.f;
        }
        // softmax_R backward of the region-attention input: dz_k = p_k (g_k - sum_j g_j p_j).  The region channels of din are
        // read only here, once the logits are dead, which keeps the kernel in registers.
        if (ATT && din_hi != nullptr) {
            constexpr int RO = W2D ? 5 : 3;
            float mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) mx = k < nreg ? fmaxf(mx, z[MO + 4 + k]) : mx;
            float s = 0.f, dot = 0.f;
            float pk[kNumReg];
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) {
                pk[k] = k < nreg ? expf(z[MO + 4 + k] - mx) : 0.f;
                s += pk[k];
            }
            load_din(din_hi, din_lo, pix, pnp_ld, gin, 72);
            if (DB) {
                const float f = (float)__ldg(keep + pix) * db_scale;
#pragma unroll
                for (int k = 0; k < 72; ++k) gin[k] *= f;
            }
            const float inv = 1.f / s;
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) {
                pk[k] *= inv;
                dot = k < nreg ? fmaf(gin[RO + k], pk[k], dot) : dot;
            }
#pragma unroll
            for (int k = 0; k < kNumReg; ++k) d[MO + 4 + k] = k < nreg ? d[MO + 4 + k] + pk[k] * (gin[RO + k] - dot) : 0.f;
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

static inline int px_grid(long total) {
    long g = (total + 127) / 128;
    const long cap = (long)num_sms() * 16;
    return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

// (mask_loss, mask_out) pairs the head can have: L1 and BCE with one mask logit, CE with two
static inline int check_mask_head(const char* fn, int mask_loss, int mask_out) {
    const bool ok = (mask_loss == kMaskL1 && mask_out == 1) || (mask_loss == kMaskBCE && mask_out == 1) ||
                    (mask_loss == kMaskCE && mask_out == 2);
    return ok ? 0 : set_error(GDRN_ERR_ARG, "%s: unsupported mask head (mask_loss %d, mask_out %d)", fn, mask_loss, mask_out);
}

static inline int check_regions(const char* fn, int num_regions, int region_att, int pnp_ld) {
    if (num_regions < 2 || num_regions > kNumReg)
        return set_error(GDRN_ERR_ARG, "%s: num_regions %d unsupported (2..64)", fn, num_regions);
    if (region_att != 0 && region_att != 1) return set_error(GDRN_ERR_ARG, "%s: region_att %d (0 or 1)", fn, region_att);
    if (pnp_ld != 64 && pnp_ld != 128) return set_error(GDRN_ERR_ARG, "%s: pnp_ld %d (64 or 128)", fn, pnp_ld);
    return 0;
}

// the Patch-PnP input width must be round_up(nIn, 64), nIn = 3 (+2 with_2d) (+num_regions with attention)
static inline int check_pnp_ld(const char* fn, int with_2d, int num_regions, int region_att, int pnp_ld) {
    const int nin = 3 + (with_2d ? 2 : 0) + (region_att ? num_regions : 0);
    if (pnp_ld != (nin + 63) / 64 * 64)
        return set_error(GDRN_ERR_ARG, "%s: pnp_ld %d for a %d-channel Patch-PnP input (want %d)", fn, pnp_ld, nin, (nin + 63) / 64 * 64);
    return 0;
}

}  // namespace gdrn
