// DropBlock on the Patch-PnP input (PNP_NET.PNP_HEAD_CFG.drop_prob / dropblock_size; conv_pnp_net.py:66-72,128-142,
// core/utils/dropblock/{dropblock,scheduler}.py):
//
//   schedule   LinearScheduler(start 0, stop drop_prob, 5000 steps): forward k (counted from 0) uses np.linspace(0, drop_prob,
//              5000)[min(k, 4999)]; every forward advances k, in train and in eval mode
//   seeds      torch.rand(B, H, W) < gamma, gamma = p / block_size^2 rounded to float32: one draw per (crop, pixel)
//   block mask keep = 1 - max_pool2d(seeds, block_size, stride 1, padding block_size / 2) (an even size crops the last row and
//              column); train mode only, and p = 0 keeps everything
//   scaling    out = x * keep * numel / sum(keep), the sum over the whole batch
//
// gdrn_dropblock_step samples the block mask on the device: the step counter k lives in device memory and is read and
// incremented by the kernels, so a captured CUDA graph draws a fresh mask at every replay.  The random numbers are
// counter-based Philox4x32-10, key (seed, rank), counter (pixel quad, crop, k): the same seed gives the same sequence.
// The glue, stand-alone packing and head-backward kernels of pixel_head.cuh apply keep * scale with their DB flag set
// (the _db entry points below).
#include <curand_philox4x32_x.h>

#include "pixel_head.cuh"

namespace gdrn {

constexpr int kDbMaxSide = 64;    // H, W <= 64: a crop's seed and row-dilation maps fit in 2 x 4 KB of shared memory
constexpr int kDbSteps = 5000;    // LinearScheduler nr_steps

// np.linspace(0, p, 5000)[min(k, 4999)] bit for bit: i * (p / 4999) in float64 (numpy divides first, then multiplies; a
// zero step means (i / 4999) * p), the last value exactly p
__device__ __forceinline__ double dropblock_prob(double p, long long k) {
    if (k >= kDbSteps - 1) return p;
    const double i = (double)k;
    const double step = p / (double)(kDbSteps - 1);
    return step == 0.0 ? (i / (double)(kDbSteps - 1)) * p : i * step;
}

// One CTA per crop: seeds (Philox, 4 pixels per draw), the k x k dilation as a row pass and a column pass in shared memory,
// the keep bytes, and the crop's kept count.
__global__ void __launch_bounds__(256) dropblock_sample_kernel(const long long* __restrict__ step, uint2 key, double p, int bs,
                                                               uint8_t* __restrict__ keep, uint8_t* __restrict__ seeds,
                                                               int* __restrict__ counts, int H, int W) {
    __shared__ uint8_t s_seed[kDbMaxSide * kDbMaxSide];
    __shared__ uint8_t s_row[kDbMaxSide * kDbMaxSide];
    __shared__ int s_cnt[8];
    const int b = blockIdx.x, HW = H * W, pad = bs / 2;
    const long long k = __ldg(step);
    const float gamma = (float)(dropblock_prob(p, k) / (double)(bs * bs));
    const long long base = (long long)b * HW;
    for (int q = threadIdx.x; q < (HW + 3) / 4; q += blockDim.x) {
        const uint4 r = curand_Philox4x32_10(make_uint4((unsigned)q, (unsigned)b, (unsigned)k, (unsigned)(k >> 32)), key);
        const unsigned rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int hw = 4 * q + j;
            if (hw < HW) {
                const uint8_t sd = (float)(rr[j] >> 8) * (1.f / 16777216.f) < gamma;  // uniform on [0, 1) in steps of 2^-24
                s_seed[hw] = sd;
                seeds[base + hw] = sd;
            }
        }
    }
    __syncthreads();
    for (int hw = threadIdx.x; hw < HW; hw += blockDim.x) {
        const int y = hw / W, x = hw - y * W;
        uint8_t any = 0;
        for (int t = 0; t < bs; ++t) {
            const int xx = x - pad + t;
            any |= (xx >= 0 && xx < W) ? s_seed[y * W + xx] : (uint8_t)0;
        }
        s_row[hw] = any;
    }
    __syncthreads();
    int kept = 0;
    for (int hw = threadIdx.x; hw < HW; hw += blockDim.x) {
        const int y = hw / W, x = hw - y * W;
        uint8_t any = 0;
        for (int t = 0; t < bs; ++t) {
            const int yy = y - pad + t;
            any |= (yy >= 0 && yy < H) ? s_row[yy * W + x] : (uint8_t)0;
        }
        keep[base + hw] = !any;
        kept += !any;
    }
    for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
    if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = kept;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += s_cnt[w];
        counts[b] = s;
    }
}

// scale = numel / sum(keep) from the per-crop counts (integer sums: exact in any order), then k += 1.  B = 0: only k += 1.
__global__ void dropblock_finish_kernel(long long* __restrict__ step, const int* __restrict__ counts, float* __restrict__ scale,
                                        int B, int HW) {
    if (threadIdx.x != 0) return;
    if (B > 0) {
        long long s = 0;
        for (int b = 0; b < B; ++b) s += counts[b];
        *scale = __fdiv_rn((float)((long long)B * HW), (float)s);
    }
    *step += 1;
}

}  // namespace gdrn

using namespace gdrn;

extern "C" int gdrn_dropblock_step(long long* step, long long seed, int rank, double drop_prob, int block_size, int train,
                                   unsigned char* keep, unsigned char* seeds, int* counts, float* scale, int B, int H, int W,
                                   void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (step == nullptr) return set_error(GDRN_ERR_ARG, "dropblock_step: step counter missing");
    if (!(drop_prob >= 0.0 && drop_prob <= 1.0))
        return set_error(GDRN_ERR_ARG, "dropblock_step: drop_prob %g outside [0, 1]", drop_prob);
    if (block_size < 1 || block_size > 15)
        return set_error(GDRN_ERR_ARG, "dropblock_step: block_size %d unsupported (1..15)", block_size);
    if (H < 1 || H > kDbMaxSide || W < 1 || W > kDbMaxSide)
        return set_error(GDRN_ERR_ARG, "dropblock_step: %d x %d map unsupported (width and height 1..%d)", H, W, kDbMaxSide);
    if (train) {
        if (B < 1 || (long long)B * H * W >= (1LL << 24))
            return set_error(GDRN_ERR_ARG, "dropblock_step: batch %d unsupported (1 .. 2^24 pixels)", B);
        if (keep == nullptr || seeds == nullptr || counts == nullptr || scale == nullptr)
            return set_error(GDRN_ERR_ARG, "dropblock_step: keep, seeds, counts and scale are required in train mode");
        const uint2 key = make_uint2((unsigned)seed, (unsigned)((unsigned long long)seed >> 32) ^ (unsigned)rank);
        dropblock_sample_kernel<<<B, 256, 0, stream>>>(step, key, drop_prob, block_size, keep, seeds, counts, H, W);
        GDRN_CUDA_OK(cudaGetLastError());
        count_launch();
    }
    dropblock_finish_kernel<<<1, 32, 0, stream>>>(step, counts, scale, train ? B : 0, H * W);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

static int check_dropblock_args(const char* fn, const void* keep, const float* scale) {
    if (keep == nullptr || scale == nullptr) return set_error(GDRN_ERR_ARG, "%s: keep and scale are required", fn);
    return 0;
}

extern "C" int gdrn_head_glue_fwd_db(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo,
                                     int B, int HW, int with_2d, int mask_out, int num_regions, int region_att, int pnp_ld,
                                     const unsigned char* keep, const float* scale, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (int rc = check_regions("head_glue_fwd_db", num_regions, region_att, pnp_ld)) return rc;
    if (int rc = check_pnp_ld("head_glue_fwd_db", with_2d, num_regions, region_att, pnp_ld)) return rc;
    if (int rc = check_dropblock_args("head_glue_fwd_db", keep, scale)) return rc;
    if (with_2d && coord2d == nullptr) return set_error(GDRN_ERR_ARG, "head_glue_fwd_db: with_2d needs coord2d");
    if (mask_out != 1 && mask_out != 2) return set_error(GDRN_ERR_ARG, "head_glue_fwd_db: mask_out %d (1 or 2)", mask_out);
    const int grid = px_grid((long)B * HW);
#define GLUE(MO, W2D, ATT)                                                                                                  \
    head_glue_fwd2_kernel<MO, W2D, ATT, true><<<grid, 128, 0, stream>>>(logits, coord2d, extents, (bf16*)out_hi,            \
                                                                        (bf16*)out_lo, B, HW, num_regions, pnp_ld, keep, scale)
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

extern "C" int gdrn_pnp_pack_input_db(const float* coor_feat, int c_feat, const float* region, int c_reg, const float* extents,
                                      void* out_hi, void* out_lo, int B, int HW, int pnp_ld, const unsigned char* keep,
                                      const float* scale, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (c_feat < 0 || c_reg < 0 || c_feat + c_reg > 72 || c_feat + c_reg < 1)
        return set_error(GDRN_ERR_ARG, "pnp_pack_input_db: %d + %d channels unsupported (1..72)", c_feat, c_reg);
    if (pnp_ld != (c_feat + c_reg + 63) / 64 * 64)
        return set_error(GDRN_ERR_ARG, "pnp_pack_input_db: pnp_ld %d for %d channels (want %d)", pnp_ld, c_feat + c_reg,
                         (c_feat + c_reg + 63) / 64 * 64);
    if (int rc = check_dropblock_args("pnp_pack_input_db", keep, scale)) return rc;
    if (c_reg > 0 && region == nullptr) return set_error(GDRN_ERR_ARG, "pnp_pack_input_db: region missing");
    pnp_pack_input2_kernel<true><<<px_grid((long)B * HW), 128, 0, stream>>>(coor_feat, c_feat, region, c_reg, extents,
                                                                           (bf16*)out_hi, (bf16*)out_lo, B, HW, pnp_ld, keep, scale);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

template <int MODE, int MO, bool SEP>
static void head_bwd_db_launch(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_tgt, const float* m_reg,
                               const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                               const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, int nreg, int att,
                               int pnp_ld, const uint8_t* keep, const float* scale, cudaStream_t stream) {
    const int grid = px_grid((long)B * HW);
#define HB2(W2D, ATT)                                                                                                         \
    head_bwd2_kernel<MODE, MO, SEP, W2D, ATT, true><<<grid, 128, 0, stream>>>(                                                 \
        logits, gt_xyz, m_xyz, m_tgt, m_reg, labels, sums, gw, (const bf16*)din_hi, (const bf16*)din_lo, extents, (bf16*)out_hi, \
        (bf16*)out_lo, B, HW, nreg, pnp_ld, keep, scale)
    if (with_2d) {
        if (att) HB2(true, true);
        else HB2(true, false);
    } else {
        if (att) HB2(false, true);
        else HB2(false, false);
    }
#undef HB2
}

extern "C" int gdrn_head_bwd_db(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                                const float* m_region, const long long* labels, const double* sums, const float* gw,
                                const void* din_hi, const void* din_lo, const float* extents, void* out_hi, void* out_lo, int B,
                                int HW, int with_2d, int mask_loss, int mask_out, int num_regions, int region_att, int pnp_ld,
                                const unsigned char* keep, const float* scale, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (int rc = check_mask_head("head_bwd_db", mask_loss, mask_out)) return rc;
    if (int rc = check_regions("head_bwd_db", num_regions, region_att, pnp_ld)) return rc;
    if (int rc = check_pnp_ld("head_bwd_db", with_2d, num_regions, region_att, pnp_ld)) return rc;
    if (int rc = check_dropblock_args("head_bwd_db", keep, scale)) return rc;
    const bool sep = m_region != m_xyz;
#define HB(MODE, MO, SEP)                                                                                                      \
    head_bwd_db_launch<MODE, MO, SEP>(logits, gt_xyz, m_xyz, m_mask, m_region, labels, sums, gw, din_hi, din_lo, extents, out_hi, \
                                      out_lo, B, HW, with_2d, num_regions, region_att, pnp_ld, keep, scale, stream)
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
