// Parameters of the implicit-GEMM forward kernel (gemm_fwd.cu) and its epilogue (gemm_epilogue.cuh).
#pragma once
#include <cuda.h>

namespace gdrn {

// flag bit of the `act` argument of gdrn_conv_fwd / gdrn_gemm_fwd / gdrn_conv_dgrad_s2: `stats` is double [2][N]
constexpr int kActStatsF64 = 16;

struct GemmParams {
    CUtensorMap tmA[2][4];  // [plane hi/lo][stride-2 phase]
    CUtensorMap tmB[2];     // [plane hi/lo]
    int mode;               // 0 = plain 2-D GEMM, 1 = conv (4-D boxes)
    int M, N;               // valid rows / cols
    int num_m_tiles, num_n_tiles, num_kb;
    int cchunks, KW, pad, stride;
    int tiles_per_img, TH, TN;
    void* out_hi;
    void* out_lo;
    float* out_f32;
    int ldc;
    const float* bias;
    const void* res_hi;  // optional residual [rows][ldc] (16-bit planes like the output) added before the activation:
    const void* res_lo;  // the eval-mode folded conv + BN + (identity) + ReLU epilogue of a BasicBlock's second conv
    int act;       // 0 none, 1 LeakyReLU(0.1), 2 ReLU
    float* stats;  // [2][N]: sum, sum of squares (accumulated with atomics) or nullptr
    int stats_f64; // stats points to double [2][N] (the act argument's GDRN_ACT_STATS_F64 bit): the CTAs' partial sums are added
                   // in double, so the result no longer depends on the order of the atomics beyond fp32 rounding of each partial
    // Stride-2 dgrad by output-parity phases (mode 1, nphase > 0): rows index the (n, i, j) lattice of dY; phase ph writes
    // output pixel (2i + ph_a, 2j + ph_b) and sums taps [ph_tap0[ph], ph_tap0[ph+1]) of the tables below
    // (dY offset (tap_dh, tap_dw); tap_w = tap slot of the packed weight matrix).  Tiles are enumerated phase-major.
    int nphase;
    int ph_tap0[5];
    int ph_a[4], ph_b[4];
    signed char tap_dh[16], tap_dw[16], tap_w[16];  // 16 = the four 2x2-tap phases of k = 4
    int pw_log2, ph_log2;  // log2 of the dY width / height
    // Grouped variant (gemm_fwd_grouped_kernel only): output rows [g * rows_per_group, (g + 1) * rows_per_group) use weight rows
    // [group[g] * w_group_rows, ...) and bias + group[g] * bias_stride; group[g] is clamped to [0, num_w_groups).
    const int* group;
    int rows_per_group, w_group_rows, num_w_groups, bias_stride;
    // TMA-stored output (gemm_fwd_tma_kernel, chosen by the host when out_tma is set): the 16-bit planes [plane hi/lo] as
    // [M][min(ldc, N rounded up to 32)] with {64, 64} boxes
    int out_tma;
    CUtensorMap tmC[2];
};

}  // namespace gdrn
