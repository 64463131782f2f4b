// Layout conversion kernels (HBM-bound, coalesced on the destination side):
//   * fp32 OIHW / IOHW / [N][K] parameters  ->  K-major bf16 (hi, lo) GEMM operands
//   * fp32 split-K weight-gradient workspace ->  fp32 gradients in the reference's parameter layout
//   * NCHW fp32 input crops                 ->  im2col matrix of the 7x7/2 stem (bf16 hi, lo)
// Parameter layouts follow the reference state_dict (SURVEY.md 8b): Conv2d OIHW, ConvTranspose2d
// IOHW (cdpn_rot_head_region.py:82-91), Linear [out][in] with fc1's input flattened from NCHW
// (conv_pnp_net.py:145).
#include <cuda_fp16.h>
#include <stdlib.h>

#include "gdrn_internal.h"
#include "ptx.cuh"

namespace gdrn {

// dst[o][tap * ipad + i] = src[o*so + i*si + r'*sr + s'*ss],  zero for i >= I, o >= O or columns >= taps*ipad
__global__ void pack_weight_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst_hi,
                                   __nv_bfloat16* __restrict__ dst_lo, int O, int I, int KH, int KW, int opad, int ipad,
                                   int krow, long so, long si, long sr, long ss, int flip) {
    const long total = (long)opad * krow;
    for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const int o = (int)(idx / krow);
        const int col = (int)(idx - (long)o * krow);
        const int tap = col / ipad;
        const int i = col - tap * ipad;
        float v = 0.f;
        if (o < O && i < I && tap < KH * KW) {
            int r = tap / KW, s = tap - (tap / KW) * KW;
            if (flip) {
                r = KH - 1 - r;
                s = KW - 1 - s;
            }
            v = __ldg(src + o * so + i * si + r * sr + s * ss);
        }
        uint16_t h, l;
        split1(v, h, l);
        reinterpret_cast<uint16_t*>(dst_hi)[idx] = h;
        if (dst_lo != nullptr) reinterpret_cast<uint16_t*>(dst_lo)[idx] = l;
    }
}

// All per-step weight re-packs of the network in ONE launch: a device-resident job table (built once by the host,
// pointers are stable) replaces ~100 tiny launches.  Jobs are padded to multiples of 256 elements so that each block
// belongs to exactly one job (one binary search per block).
struct PackJob {
    const float* src;
    __nv_bfloat16* dst_hi;
    __nv_bfloat16* dst_lo;
    long so, si, sr, ss;
    long elem_begin;  // prefix sum of the job's tile counts: ceil(opad/16) * ceil(ipad/64) * ceil(taps/9)
    int O, I, KH, KW, opad, ipad, krow, flip;
    const float* row_scale;  // optional [O]: dst row o is multiplied by row_scale[o] -- the eval-mode BatchNorm scale
                             // gamma / sqrt(running_var + eps) folded into the conv weights (NS-1: folded conv+BN+ReLU)
};

constexpr int kPackDR = 16;  // dst rows per tile
constexpr int kPackDC = 64;  // dst channels per tile (128 bytes of one dst row segment)
constexpr int kPackTC = 9;   // taps per tile
constexpr int kPackLD = kPackDC + 1;

__global__ void __launch_bounds__(256) pack_weight_batched_kernel(const PackJob* __restrict__ jobs, int njobs, long total_blocks) {
    pdl_ew_entry();
    // One block = one tile of 16 dst rows x 64 dst channels x <= 9 taps, staged through shared memory:
    //   load : threads walk the tile in SOURCE order (taps innermost, then whichever of the row / channel strides is
    //          smaller), so a warp reads runs of >= 36..1152 contiguous bytes of the fp32 parameter;
    //   store: 8 threads write the 128-byte (row, tap) segment of each plane with 16-byte stores.
    // (The previous version had one thread per (row, channel) pair looping over the taps: 4-byte loads with a 36-byte
    // lane stride and 2-byte stores -- 374 us per step for 360 MB of traffic.)
    __shared__ PackJob job;
    __shared__ float tile[kPackDR * kPackTC * kPackLD];
    __shared__ int tapoff[kPackTC];
    for (long blk = blockIdx.x; blk < total_blocks; blk += gridDim.x) {
        __syncthreads();
        if (threadIdx.x == 0) {
            int lo = 0, hi = njobs - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (jobs[mid].elem_begin <= blk) lo = mid; else hi = mid - 1;
            }
            job = jobs[lo];
        }
        __syncthreads();
        const int taps = job.KH * job.KW;
        const int n_tc = (taps + kPackTC - 1) / kPackTC;
        const int n_dc = (job.ipad + kPackDC - 1) / kPackDC;
        int t = (int)(blk - job.elem_begin);  // elem_begin counts TILES
        const int tc = t % n_tc;
        t /= n_tc;
        const int dcb = t % n_dc;
        const int drb = t / n_dc;
        const int t0 = tc * kPackTC, tcn = min(kPackTC, taps - t0);
        const int dr0 = drb * kPackDR, dc0 = dcb * kPackDC;
        if (threadIdx.x < tcn) {
            int tap = t0 + threadIdx.x;
            if (job.flip) tap = taps - 1 - tap;
            const int r = tap / job.KW, s2 = tap - r * job.KW;
            tapoff[threadIdx.x] = (int)(r * job.sr + s2 * job.ss);
        }
        __syncthreads();
        const float inv_tcn = 1.f / (float)tcn;
        const bool chan_fast = job.si <= job.so;  // consecutive source addresses: (tap, channel, row) or (tap, row, channel)
        for (int f = threadIdx.x; f < kPackDR * kPackDC * tcn; f += 256) {
            const int q = __float2int_rd(((float)f + 0.5f) * inv_tcn);
            const int tl = f - q * tcn;
            const int dc = chan_fast ? (q % kPackDC) : (q / kPackDR);
            const int dr = chan_fast ? (q / kPackDC) : (q % kPackDR);
            const int o = dr0 + dr, i = dc0 + dc;
            float v = 0.f;
            if (o < job.O && i < job.I) {
                v = __ldg(job.src + o * job.so + i * job.si + tapoff[tl]);
                if (job.row_scale != nullptr) v *= __ldg(job.row_scale + o);
            }
            tile[(dr * kPackTC + tl) * kPackLD + dc] = v;
        }
        __syncthreads();
        uint16_t* dh = reinterpret_cast<uint16_t*>(job.dst_hi);
        uint16_t* dl = reinterpret_cast<uint16_t*>(job.dst_lo);
        if ((job.ipad & 7) == 0 && (job.krow & 7) == 0) {
            for (int it = threadIdx.x; it < kPackDR * tcn * (kPackDC / 8); it += 256) {
                const int g = it & 7, row = it >> 3;
                const int dr = __float2int_rd(((float)row + 0.5f) * inv_tcn);
                const int tl = row - dr * tcn;
                const int o = dr0 + dr, i = dc0 + g * 8;
                if (o >= job.opad || i >= job.ipad) continue;
                const float* src = tile + (dr * kPackTC + tl) * kPackLD + g * 8;
                uint4 h, l;
                split2(src[0], src[1], h.x, l.x);
                split2(src[2], src[3], h.y, l.y);
                split2(src[4], src[5], h.z, l.z);
                split2(src[6], src[7], h.w, l.w);
                const long off = (long)o * job.krow + (long)(t0 + tl) * job.ipad + i;
                *reinterpret_cast<uint4*>(dh + off) = h;
                if (dl != nullptr) *reinterpret_cast<uint4*>(dl + off) = l;
            }
        } else {  // odd channel padding (the 7x7 stem: 3 channels per tap): scalar stores
            for (int it = threadIdx.x; it < kPackDR * tcn * kPackDC; it += 256) {
                const int dc = it & (kPackDC - 1), row = it / kPackDC;
                const int dr = __float2int_rd(((float)row + 0.5f) * inv_tcn);
                const int tl = row - dr * tcn;
                const int o = dr0 + dr, i = dc0 + dc;
                if (o >= job.opad || i >= job.ipad) continue;
                uint16_t h, l;
                split1(tile[(dr * kPackTC + tl) * kPackLD + dc], h, l);
                const long off = (long)o * job.krow + (long)(t0 + tl) * job.ipad + i;
                dh[off] = h;
                if (dl != nullptr) dl[off] = l;
            }
        }
    }
}

// grad[o*so + i*si + r'*sr + s'*ss] (+)= sum_ks ws[ks][o*krow + tap*ipad + i]
//
// One block per (output row o, chunk of IC input channels): the split-K partial sums are read with KP-way parallelism
// over the splits (coalesced over i, 4 independent loads in flight per thread), reduced through shared memory, transposed
// there from the workspace's (tap, i) order to the parameter's (i, tap) order and written out as one contiguous run
// (Conv2d OIHW: IC*taps floats).  The first version (one thread per element, serial loop over the splits, 36-byte-strided
// stores) was latency-bound: 50-150 us for layers whose whole workspace is a few MB.
template <int VARIANT>
__global__ void __launch_bounds__(256) unpack_wgrad_kernel(const float* __restrict__ ws, float* __restrict__ grad, int O, int I,
                                                           int KH, int KW, int IC, int n_ic, int KP, int ipad, int krow_,
                                                           int ksplit, long ks_stride, long so, long si, long sr, long ss,
                                                           int flip, int accumulate) {
    pdl_ew_entry();
    extern __shared__ __align__(16) float sm[];
    const int taps = KH * KW;
    const int nelem = taps * IC;
    const int tstride = taps | 1;  // odd: conflict-free transposed stores
    float* red = sm;               // [KP][nelem]
    float* out = sm + KP * nelem;  // [IC][tstride]
    const int o = blockIdx.x / n_ic;
    const int i0 = (blockIdx.x - o * n_ic) * IC;
    const int icn = min(IC, I - i0);
    const float inv_nelem = 1.f / (float)nelem, inv_ic = 1.f / (float)IC, inv_taps = 1.f / (float)taps;
    const float* base = ws + (long)o * krow_ + i0;
    const long kstep = (long)KP * ks_stride;
    if (VARIANT == 1) {  // scalar loads: shapes whose rows are not 16-byte aligned (the 7x7 stem, 3 channels per tap)
        for (int item = threadIdx.x; item < KP * nelem; item += 256) {
            const int kp = __float2int_rd(((float)item + 0.5f) * inv_nelem);
            const int e = item - kp * nelem;
            const int tap = __float2int_rd(((float)e + 0.5f) * inv_ic);
            const int i = e - tap * IC;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            if (i < icn) {
                const float* sp = base + (long)tap * ipad + i + (long)kp * ks_stride;
                int ks = kp;
                for (; ks + 3 * KP < ksplit; ks += 4 * KP) {
                    a0 += sp[0];
                    a1 += sp[kstep];
                    a2 += sp[2 * kstep];
                    a3 += sp[3 * kstep];
                    sp += 4 * kstep;
                }
                for (; ks < ksplit; ks += KP) {
                    a0 += *sp;
                    sp += kstep;
                }
            }
            red[item] = (a0 + a1) + (a2 + a3);
        }
    } else {
        // 16-byte loads (IC, ipad, krow and the split stride are multiples of 4 floats -- checked by the host): with one
        // request per thread in flight, 4-byte loads cap an SM at ~8 KB outstanding (~1.5 TB/s of L2 reads over 132 SMs).
        const int ic4 = IC >> 2;
        const int nvec = taps * ic4;
        const float inv_nvec = 1.f / (float)nvec, inv_ic4 = 1.f / (float)ic4;
        const long kstep4 = kstep >> 2;
#pragma unroll 2
        for (int item = threadIdx.x; item < KP * nvec; item += 256) {
            const int kp = __float2int_rd(((float)item + 0.5f) * inv_nvec);
            const int e4 = item - kp * nvec;
            const int tap = __float2int_rd(((float)e4 + 0.5f) * inv_ic4);
            const int i = (e4 - tap * ic4) * 4;
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < icn) {  // icn is a multiple of 4 here
                const float4* sp = reinterpret_cast<const float4*>(base + (long)tap * ipad + i + (long)kp * ks_stride);
                int ks = kp;
                for (; ks + KP < ksplit; ks += 2 * KP) {
                    const float4 v0 = __ldg(sp), v1 = __ldg(sp + kstep4);
                    a.x += v0.x; a.y += v0.y; a.z += v0.z; a.w += v0.w;
                    b.x += v1.x; b.y += v1.y; b.z += v1.z; b.w += v1.w;
                    sp += 2 * kstep4;
                }
                if (ks < ksplit) {
                    const float4 v0 = __ldg(sp);
                    a.x += v0.x; a.y += v0.y; a.z += v0.z; a.w += v0.w;
                }
            }
            float* r = red + kp * nelem + tap * IC + i;
            *reinterpret_cast<float4*>(r) = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nelem; e += 256) {
        float v = red[e];
        for (int kp = 1; kp < KP; ++kp) v += red[kp * nelem + e];
        const int tap = __float2int_rd(((float)e + 0.5f) * inv_ic);
        const int i = e - tap * IC;
        out[i * tstride + (flip ? taps - 1 - tap : tap)] = v;
    }
    __syncthreads();
    float* gbase = grad + (long)o * so + (long)i0 * si;
    for (int j = threadIdx.x; j < icn * taps; j += 256) {
        const int i = __float2int_rd(((float)j + 0.5f) * inv_taps);
        const int tp = j - i * taps;
        const int r = tp / KW, s = tp - r * KW;
        float* d = gbase + (long)i * si + r * sr + s * ss;
        const float v = out[i * tstride + tp];
        *d = accumulate ? (*d + v) : v;
    }
}

// Stem im2col: x NCHW fp32 [B,3,H,W] -> A[(b,oh,ow)][192] with k = (r*7+s)*3 + c (147 valid), conv 7x7 s2 p3.
// One block per (image, output row): the 7 x 3 input rows it needs are staged in shared memory with a zero halo
// (coalesced fp32 loads), then every thread emits 16-byte groups of 8 consecutive k for consecutive positions
// (coalesced stores; the matrix is 403 MB per plane at B=64, so the stores are what matters).
template <int W>
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ a_hi,
                                                          __nv_bfloat16* __restrict__ a_lo, int B, int H) {
    pdl_ew_entry();
    constexpr int WP = W + 6;  // 3-pixel zero halo left and right
    __shared__ float tile[3][7][WP];
    const int Ho = H / 2, Wo = W / 2;
    const int b = blockIdx.x / Ho, oh = blockIdx.x - b * Ho;
    for (int e = threadIdx.x; e < 3 * 7 * WP; e += 256) {
        const int col = e % WP;
        const int r = (e / WP) % 7;
        const int c = e / (WP * 7);
        const int ih = oh * 2 + r - 3, iw = col - 3;
        float v = 0.f;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(x + (((long)b * 3 + c) * H + ih) * W + iw);
        tile[c][r][col] = v;
    }
    __syncthreads();
    const long row0 = ((long)b * Ho + oh) * Wo;
    // thread = (k-group g of 8 consecutive k, lane l over output columns): the eight (c, r, s) tile offsets of a group are
    // computed ONCE (the first version redid two integer divisions per element: ALU-bound at 2.3x the store time); a warp
    // still writes 32 consecutive 16-byte groups = 512 contiguous bytes per plane.
    if (threadIdx.x < 240) {
        const int g = threadIdx.x % 24, l = threadIdx.x / 24;
        int off[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = g * 8 + j;
            if (k < 147) {
                const int tap = k / 3, c = k - tap * 3;
                const int r = tap / 7, s2 = tap - r * 7;
                off[j] = (c * 7 + r) * WP + s2;
            } else {
                off[j] = -1;
            }
        }
        const float* tf = &tile[0][0][0];
        for (int ow = l; ow < Wo; ow += 10) {
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = off[j] >= 0 ? tf[off[j] + 2 * ow] : 0.f;
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                split2(v[2 * j], v[2 * j + 1], hi[j], lo[j]);
            }
            const long idx = (row0 + ow) * 24 + g;
            reinterpret_cast<uint4*>(a_hi)[idx] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            if (a_lo != nullptr) reinterpret_cast<uint4*>(a_lo)[idx] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
    }
}

static inline int grid_for(long total, int block) {
    long g = (total + block - 1) / block;
    const long cap = (long)num_sms() * 16;
    return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

}  // namespace gdrn

using namespace gdrn;

extern "C" int gdrn_pack_weight(const float* src, void* dst_hi, void* dst_lo, int O, int I, int KH, int KW, int opad,
                                int ipad, int krow, long so, long si, long sr, long ss, int flip, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (krow < KH * KW * ipad || opad < O || ipad < I) return set_error(GDRN_ERR_ARG, "pack_weight: bad padding");
    const long total = (long)opad * krow;
    pack_weight_kernel<<<grid_for(total, 256), 256, 0, stream>>>(src, (__nv_bfloat16*)dst_hi, (__nv_bfloat16*)dst_lo, O, I,
                                                                KH, KW, opad, ipad, krow, so, si, sr, ss, flip);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_unpack_wgrad(const float* ws, float* grad, int O, int I, int KH, int KW, int ipad, int krow, int ksplit,
                                 long ks_stride, long so, long si, long sr, long ss, int flip, int accumulate,
                                 void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const int taps = KH * KW;
    if (O <= 0 || I <= 0 || taps <= 0 || ksplit <= 0) return set_error(GDRN_ERR_ARG, "unpack_wgrad: empty shape");
    // tile: all taps x IC channels of one output row.  IC grows (32 -> 256) until a block has >= 512 sixteen-byte loads to
    // issue (few-split layers such as 512->512 would otherwise run thousands of blocks with 144 busy threads each);
    // the split-K partials of a tile are staged in <= 32 KB of shared memory, KP = ways of parallelism over the splits.
    int IC = taps == 1 ? 256 : 32, KP = 1, nelem = 0;
    if (IC > I) IC = I;
    while (taps * IC > 2048 && IC > 1) IC >>= 1;
    for (;;) {
        nelem = taps * IC;
        KP = 8192 / nelem;
        if (KP > 16) KP = 16;
        if (KP > ksplit) KP = ksplit;
        if (KP < 1) KP = 1;
        if (KP * nelem / 4 >= 512 || IC * 2 > I || IC * 2 > 256 || taps * IC * 2 > 2304) break;
        IC *= 2;
    }
    if (nelem > 2304) return set_error(GDRN_ERR_ARG, "unpack_wgrad: kernel window too large");
    const int n_ic = (I + IC - 1) / IC;
    const size_t smem = ((size_t)KP * nelem + (size_t)IC * (taps | 1)) * sizeof(float);
    static int variant = -1;
    if (variant < 0) {
        const char* e = getenv("GDRN_UNPACK");
        variant = e ? atoi(e) : 0;
    }
    const bool vec_ok = (IC % 4 == 0) && (I % 4 == 0) && (ipad % 4 == 0) && (krow % 4 == 0) && (ks_stride % 4 == 0) &&
                        ((reinterpret_cast<uintptr_t>(ws) & 15) == 0);
    if (variant == 1 || !vec_ok)
        GDRN_LAUNCH_PDL(unpack_wgrad_kernel<1>, O * n_ic, 256, smem, stream, ws, grad, O, I, KH, KW, IC, n_ic, KP, ipad, krow, ksplit, ks_stride,
                                                               so, si, sr, ss, flip, accumulate);
    else
        GDRN_LAUNCH_PDL(unpack_wgrad_kernel<0>, O * n_ic, 256, smem, stream, ws, grad, O, I, KH, KW, IC, n_ic, KP, ipad, krow, ksplit, ks_stride,
                                                               so, si, sr, ss, flip, accumulate);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_stem_im2col(const float* x, void* a_hi, void* a_lo, int B, int H, int W, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (H % 2 || W != 256) return set_error(GDRN_ERR_ARG, "stem_im2col: expects 256-wide crops (INPUT_RES=256), even height");
    GDRN_LAUNCH_PDL_FWD(stem_im2col_kernel<256>, B * (H / 2), 256, 0, stream, x, (__nv_bfloat16*)a_hi, (__nv_bfloat16*)a_lo, B, H);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_pack_weight_batched(const void* jobs_dev, int njobs, long total_blocks, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    static_assert(sizeof(PackJob) == 104, "PackJob layout is mirrored by the host (gdr_net_b200/engine.py)");
    if (njobs <= 0) return 0;
    long grid = total_blocks;
    const long cap = (long)num_sms() * 16;
    if (grid > cap) grid = cap;
    GDRN_LAUNCH_PDL(pack_weight_batched_kernel, (int)grid, 256, 0, stream, reinterpret_cast<const PackJob*>(jobs_dev), njobs, total_blocks);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
