// Tile epilogue of the implicit-GEMM forward kernel (gemm_fwd.cu), run by each MMA warpgroup on its 64 x BLOCK_N register
// accumulators: bias -> residual -> activation -> 16-bit hi[/lo] and / or fp32
// stores -> per-channel sum / sum of squares for the BatchNorm batch statistics.
#pragma once
#include "gdrn_internal.h"
#include "gemm_params.h"
#include "ptx.cuh"

namespace gdrn {

// acc    : this thread's BLOCK_N / 2 accumulator values (wgmma.cuh layout; in the 3-pass mode the cross terms are already folded in);
// row0   : row of the 128-row tile held in acc[4j + 0..1] (acc[4j + 2..3] hold row0 + 8); q = lane % 4 selects the column pair;
// s_stats: the CTA's [2][BLOCK_N] partial BatchNorm sums.
// Columns are written in 32-wide chunks like the output tiles: a chunk that starts at or beyond N is left untouched, inside a
// partial chunk the columns in [N, ldc) are zero-filled.
// The only per-row state kept across the unrolled column loop is one 32-bit element offset (and a validity flag) per row,
// shared by the output and residual planes; the host entry points reject outputs with rows * ldc >= 2^32.  Addresses are
// rebuilt from the kernel parameters for every chunk: unsigned arithmetic keeps the compiler from hoisting them into 64-bit
// per-row pointers, which would not fit next to the accumulators of a 128-wide 3-pass tile.
// GROUPED: the bias of this tile starts at p.bias + bias_off (the tile's weight group, gemm_fwd_grouped_kernel).
// STAGED: the 16-bit planes are not stored here but written to this warpgroup's staging area `stg` in shared memory (plane p at
//          stg + p * (J1 - J0) * 1024: one 128-byte-swizzled [64 rows][64 columns] box per 64 columns, 8 KB apart), from where
//          the kernel stores them with TMA.  fp32 outputs are always stored here.
// J0, J1 : the column groups (8 columns each) of this call; a 128-wide 3-pass tile is staged in two 64-column halves.
// PLAIN  : bias and activation only, one 16-bit plane (the 256-row tile): the residual, lo-plane, fp32-output, statistics and
//          output-parity code is not compiled in.
// Staging slot of (column group j, row half h) of this thread's first plane: row r of a box keeps its 16-byte column chunk c at
// chunk c ^ (r % 8) (SWIZZLE_128B); the 8 rows of a warp's store have distinct r % 8, so the 32 lanes hit 32 distinct banks.
__device__ __forceinline__ uint32_t* stage_slot(uint8_t* stg, int row0, int lane, int j, int h) {
    return reinterpret_cast<uint32_t*>(stg + (row0 & 63) * 128 + 4 * (lane & 3) + (j >> 3) * 8192 + (((j & 7) ^ (row0 & 7)) << 4) +
                                       h * 1024);
}

template <int BLOCK_N, bool GROUPED = false, bool STAGED = false, int J0 = 0, int J1 = BLOCK_N / 8, bool PLAIN = false>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmParams& p, const float* acc, int lane, int row0, int m_tile, int n_tile,
                                                   int ph, float* s_stats, int bias_off = 0, uint8_t* stg = nullptr) {
    static_assert(!PLAIN || STAGED, "the plain epilogue is the TMA-stored one");
    __nv_bfloat16* out_hi = reinterpret_cast<__nv_bfloat16*>(p.out_hi);
    __nv_bfloat16* out_lo = PLAIN ? nullptr : reinterpret_cast<__nv_bfloat16*>(p.out_lo);
    const __nv_bfloat16* res_hi = PLAIN ? nullptr : reinterpret_cast<const __nv_bfloat16*>(p.res_hi);
    const __nv_bfloat16* res_lo = PLAIN ? nullptr : reinterpret_cast<const __nv_bfloat16*>(p.res_lo);
    float* const out_f32 = PLAIN ? nullptr : p.out_f32;
    const int q = lane & 3;
    uint32_t off[2];  // element offset of (output row, this thread's first column) in the [rows][ldc] planes
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int mrow = m_tile * 128 + row0 + 8 * h;
        row_ok[h] = mrow < p.M;
        uint32_t grow = (uint32_t)mrow;  // output row
        if (!PLAIN && p.nphase) {  // (n, i, j) of the dY lattice -> pixel (2i + a, 2j + b) of the 2x larger dX
            const uint32_t j = grow & ((1u << p.pw_log2) - 1);
            const uint32_t t = grow >> p.pw_log2;
            const uint32_t i = t & ((1u << p.ph_log2) - 1);
            const uint32_t n = t >> p.ph_log2;
            grow = (((n << (p.ph_log2 + 1)) + 2 * i + p.ph_a[ph]) << (p.pw_log2 + 1)) + 2 * j + p.ph_b[ph];
        }
        off[h] = grow * (uint32_t)p.ldc + (uint32_t)(n_tile * BLOCK_N + 2 * q);
    }
#pragma unroll
    for (int j = J0; j < J1; ++j) {
        const int cl = 8 * j + 2 * q;  // column inside the tile
        const int col = n_tile * BLOCK_N + cl;
        if (n_tile * BLOCK_N + 32 * (j / 4) >= p.N) continue;  // warp-uniform: chunk beyond N
        const bool ok0 = col < p.N, ok1 = col + 1 < p.N;
        float f[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) f[h][e] = acc[4 * j + 2 * h + e];
        if (p.bias != nullptr) {
            // (the group offset is spelled inside each load: a hoisted bias pointer costs the ungrouped kernels registers)
            const int c0 = GROUPED ? bias_off + col : col;
            const float b0 = ok0 ? __ldg(p.bias + c0) : 0.f, b1 = ok1 ? __ldg(p.bias + c0 + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                f[h][0] += b0;
                f[h][1] += b1;
            }
        }
        if (res_hi != nullptr && ok0) {
            // folded eval epilogue: + residual (the block's identity / downsample branch, same [rows][ldc] planes; N % 32 == 0)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!row_ok[h]) continue;
                float a, b;
                unpack_hi2(__ldg(reinterpret_cast<const uint32_t*>(res_hi + (off[h] + 8 * j))), a, b);
                f[h][0] += a;
                f[h][1] += b;
                if (res_lo != nullptr) {
                    unpack_lo2(__ldg(reinterpret_cast<const uint32_t*>(res_lo + (off[h] + 8 * j))), a, b);
                    f[h][0] += a;
                    f[h][1] += b;
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (p.act == 1) f[h][e] = f[h][e] > 0.f ? f[h][e] : 0.1f * f[h][e];
                else if (p.act == 2) f[h][e] = fmaxf(f[h][e], 0.f);
            }
        if constexpr (STAGED) {
            // rows beyond M and columns beyond the output map's width are clipped by the TMA store
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float a = ok0 ? f[h][0] : 0.f, b = ok1 ? f[h][1] : 0.f;
                uint32_t* const d = stage_slot(stg, row0, lane, j - J0, h);
                uint32_t hi, lo;
                if (out_lo != nullptr) {
                    split2(a, b, hi, lo);
                    d[(J1 - J0) * 256] = lo;  // the lo plane, (J1 - J0) * 1024 bytes on
                } else {
                    hi = pack_hi2(a, b);
                }
                *d = hi;
            }
        }
        if (col < p.ldc) {  // ldc % 8 == 0: the pair (col, col + 1) is inside or outside together
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!row_ok[h]) continue;
                const float a = ok0 ? f[h][0] : 0.f, b = ok1 ? f[h][1] : 0.f;
                const uint32_t o = off[h] + 8 * j;
                if (out_f32 != nullptr) *reinterpret_cast<float2*>(out_f32 + o) = make_float2(a, b);
                if (!STAGED && out_hi != nullptr) {
                    uint32_t hi, lo;
                    if (out_lo != nullptr) {
                        split2(a, b, hi, lo);
                        *reinterpret_cast<uint32_t*>(out_lo + o) = lo;
                    } else {
                        hi = pack_hi2(a, b);
                    }
                    *reinterpret_cast<uint32_t*>(out_hi + o) = hi;
                }
            }
        }
        if (!PLAIN && p.stats != nullptr) {
            // per-channel sum / sum of squares over the warp's 16 rows: the 8 lanes sharing q hold the same two columns
            float s1[2], s2[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float v0 = row_ok[0] ? f[0][e] : 0.f, v1 = row_ok[1] ? f[1][e] : 0.f;
                s1[e] = v0 + v1;
                s2[e] = fmaf(v1, v1, v0 * v0);
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
                    s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], off);
                    s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], off);
                }
            }
            if (lane < 4) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    atomicAdd(&s_stats[cl + e], s1[e]);
                    atomicAdd(&s_stats[BLOCK_N + cl + e], s2[e]);
                }
            }
        }
    }
}

}  // namespace gdrn
