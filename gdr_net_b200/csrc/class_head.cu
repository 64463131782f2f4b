// Class-aware geometry head (ROT_HEAD.ROT_CLASS_AWARE / MASK_CLASS_AWARE / REGION_CLASS_AWARE, reference GDRN.py:134-151,
// cdpn_rot_head_region.py:114-135): the 1x1 output conv holds one block of rows per object class and every crop uses the rows
// of its own class.  The forward and the data gradient run as grouped GEMMs (gdrn_conv_fwd_grouped / gdrn_gemm_fwd_grouped,
// gemm_fwd.cu) over class-major weight tables; this file holds the table gather and the weight / bias gradient reduction.
//
//   gdrn_class_gather       dst[i][k] = src[idx[i]][k] (0 where idx[i] < 0): the class-major weight / bias tables, per step
//   gdrn_crop_colsum        per-crop column sums of the logit gradient (bias partials), fixed summation order
//   gdrn_class_wgrad_reduce grad[r] = sum over crops b in crop order of partial_b[slot(class_b, r)], 0 for rows no crop uses
#include "gdrn_internal.h"
#include "ptx.cuh"

namespace gdrn {

typedef __nv_bfloat16 bf16;

__global__ void class_gather_kernel(const float* __restrict__ src, const int* __restrict__ idx, float* __restrict__ dst, int n_dst,
                                    int K, int n_src) {
    pdl_ew_entry();
    const long total = (long)n_dst * K;
    for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const int i = (int)(e / K), k = (int)(e - (long)i * K);
        const int r = __ldg(idx + i);
        dst[e] = (r >= 0 && r < n_src) ? __ldg(src + (long)r * K + k) : 0.f;
    }
}

// One CTA per crop: 8-column groups x row lanes; the row lanes' partial sums are added in lane order.
constexpr int kColsumThreads = 512;

__global__ void __launch_bounds__(kColsumThreads) crop_colsum_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo,
                                                                   float* __restrict__ out, int rows, int ld) {
    pdl_ew_entry();
    const int cg = ld / 8, lanes = kColsumThreads / cg;
    const int g = threadIdx.x % cg, rl = threadIdx.x / cg;
    const long base = (long)blockIdx.x * rows;
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = 0.f;
    for (int r = rl; r < rows; r += lanes) {
        const long off8 = (base + r) * cg + g;
        float f[8];
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(x_hi) + off8);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) unpack_hi2(w[j], f[2 * j], f[2 * j + 1]);
        if (x_lo != nullptr) {
            const uint4 ql = __ldg(reinterpret_cast<const uint4*>(x_lo) + off8);
            const uint32_t wl[4] = {ql.x, ql.y, ql.z, ql.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float a, b;
                unpack_lo2(wl[j], a, b);
                f[2 * j] += a;
                f[2 * j + 1] += b;
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] += f[j];
    }
    __shared__ float red[kColsumThreads][8 + 1];
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x][j] = s[j];
    __syncthreads();
    for (int c = threadIdx.x; c < ld; c += kColsumThreads) {
        float a = 0.f;
        for (int q = 0; q < lanes; ++q) a += red[q * cg + c / 8][c % 8];
        out[(long)blockIdx.x * ld + c] = a;
    }
}

// One CTA per reference row r; thread k < K sums weight column k, k == K the bias.  slot_of[c][r] = the logit slot of row r for
// class c, or -1; classes are clamped to [0, num_classes) and slots checked against n_slots.
__global__ void class_wgrad_reduce_kernel(const float* __restrict__ ws, long ws_crop_stride, int ws_ld, const float* __restrict__ bias_part,
                                          int bias_ld, const int* __restrict__ classes, int B, const int* __restrict__ slot_of,
                                          int num_classes, int n_rows, int n_slots, int K, float* __restrict__ grad_w,
                                          float* __restrict__ grad_b) {
    pdl_ew_entry();
    const int r = blockIdx.x;
    for (int k = threadIdx.x; k <= K; k += blockDim.x) {
        float acc = 0.f;
        for (int b = 0; b < B; ++b) {
            const int c = min(max(__ldg(classes + b), 0), num_classes - 1);
            const int s = __ldg(slot_of + (long)c * n_rows + r);
            if (s < 0 || s >= n_slots) continue;
            acc += k < K ? __ldg(ws + b * ws_crop_stride + (long)s * ws_ld + k) : __ldg(bias_part + (long)b * bias_ld + s);
        }
        if (k < K) grad_w[(long)r * K + k] = acc;
        else grad_b[r] = acc;
    }
}

}  // namespace gdrn

using namespace gdrn;

extern "C" int gdrn_class_gather(const float* src, const int* idx, float* dst, int n_dst, int K, int n_src, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (n_dst <= 0 || K <= 0 || n_src <= 0) return set_error(GDRN_ERR_ARG, "class_gather: bad sizes n_dst=%d K=%d n_src=%d", n_dst, K, n_src);
    if (src == nullptr || idx == nullptr || dst == nullptr) return set_error(GDRN_ERR_ARG, "class_gather: NULL pointer");
    long blocks = ((long)n_dst * K + 255) / 256;
    if (blocks > (long)num_sms() * 8) blocks = (long)num_sms() * 8;
    GDRN_LAUNCH_PDL(class_gather_kernel, (int)blocks, 256, 0, stream, src, idx, dst, n_dst, K, n_src);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_crop_colsum(const void* x_hi, const void* x_lo, float* out, int B, int rows_per_crop, int ld, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (ld <= 0 || ld % 8 || ld / 8 > kColsumThreads || kColsumThreads % (ld / 8))
        return set_error(GDRN_ERR_ARG, "crop_colsum: unsupported ld=%d", ld);
    if (B <= 0 || rows_per_crop <= 0) return set_error(GDRN_ERR_ARG, "crop_colsum: bad sizes B=%d rows_per_crop=%d", B, rows_per_crop);
    if (x_hi == nullptr || out == nullptr) return set_error(GDRN_ERR_ARG, "crop_colsum: NULL pointer");
    GDRN_LAUNCH_PDL(crop_colsum_kernel, B, kColsumThreads, 0, stream, reinterpret_cast<const bf16*>(x_hi),
                    reinterpret_cast<const bf16*>(x_lo), out, rows_per_crop, ld);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int gdrn_class_wgrad_reduce(const float* ws, long ws_crop_stride, int ws_ld, const float* bias_part, int bias_ld,
                                       const int* classes, int B, const int* slot_of, int num_classes, int n_rows, int n_slots, int K,
                                       float* grad_w, float* grad_b, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (B <= 0 || num_classes <= 0 || n_rows <= 0 || K <= 0)
        return set_error(GDRN_ERR_ARG, "class_wgrad_reduce: bad sizes B=%d num_classes=%d n_rows=%d K=%d", B, num_classes, n_rows, K);
    if (n_slots <= 0 || n_slots > bias_ld || ws_ld < K || ws_crop_stride < (long)n_slots * ws_ld)
        return set_error(GDRN_ERR_ARG, "class_wgrad_reduce: partials too small (n_slots=%d bias_ld=%d ws_ld=%d ws_crop_stride=%ld)",
                         n_slots, bias_ld, ws_ld, ws_crop_stride);
    if (!ws || !bias_part || !classes || !slot_of || !grad_w || !grad_b) return set_error(GDRN_ERR_ARG, "class_wgrad_reduce: NULL pointer");
    GDRN_LAUNCH_PDL(class_wgrad_reduce_kernel, n_rows, 256, 0, stream, ws, ws_crop_stride, ws_ld, bias_part, bias_ld, classes, B,
                    slot_of, num_classes, n_rows, n_slots, K, grad_w, grad_b);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
