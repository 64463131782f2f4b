// wgmma / TMA implicit-GEMM forward kernel (sm_90a).
//
// One persistent, warp-specialised kernel serves every GEMM-shaped forward op of the GDR-Net hot
// path (reference call sites: resnet_backbone.py:69-76 convs, cdpn_rot_head_region.py:82-135,
// conv_pnp_net.py:76-80 + fc1/fc2/fc_r/fc_t :111-157) and, with flipped weights, every dgrad:
//
//   D[M = pixels][N = Cout] = sum_k A[M][K] * W[N][K]          (16-bit operands, fp32 accumulate in registers)
//
//   * A is never materialised: for a conv, each 64-wide k-block is one (tap, channel-chunk) and its
//     128x64 A tile is ONE 4-D TMA box {64 ch, Wo, TH, TN} of the NHWC activation tensor at the
//     tap-shifted coordinate; out-of-image rows/cols are zero-filled by TMA (= conv padding).
//     Stride-2 convs read from four phase sub-lattices (one tensor map per (row, col) parity);
//     stride-2 DGRADS run as four output-parity phases over the un-dilated dY (gdrn_conv_dgrad_s2).
//   * W is a K-major [Cout][KH*KW*Cin] 16-bit matrix (prepared by pack kernels), 2-D TMA boxes.
//   * Both land in shared memory in the 128-byte-swizzled K-major layout wgmma consumes.
//   * warpgroups 0 and 1 = MMA + epilogue, each owning 64 of the 128 rows of a tile (wgmma m64nNk16,
//     accumulators in registers; the epilogue in gemm_epilogue.cuh applies bias / residual / activation,
//     stores 16-bit hi[/lo] or fp32 and accumulates the per-channel BatchNorm statistics).  While the MMA
//     warpgroups run a tile's epilogue the producer already fills the stages of the next tile.  gemm_fwd_tma_kernel (every
//     launch with a 16-bit output but the phase dgrads, make_out_maps) instead stages the 16-bit planes in a shared-memory buffer
//     behind the ring and writes them with TMA stores, so the MMAs of the next tile start while the tile drains.
//     gemm_fwd_tall_kernel (large single-pass launches with a plain epilogue, pick_block_m) runs the same body on 256-row tiles.
//     Warp 8 = TMA producer.  With nine warps ptxas allots at most 168 registers per thread (three warps share one SM
//     sub-partition's register file).  A 128-wide 3-pass tile holds 128 accumulator registers (main + cross) in its main
//     loop; it fits (ptxas -v: 162 registers, no spills) because the cross accumulator is folded into the main one before
//     the epilogue and the epilogue keeps only a 32-bit element offset per row live.  The width matters for the 3-pass mode: per
//     MMA clock a k-block moves about 190 B of shared memory (wgmma operand reads + TMA writes) at 128 x 64 and about 135 B at
//     128 x 128, against 128 B/clk per SM, so the 64-wide 3-pass tile is bound by shared-memory bandwidth.
//   * NSPLIT = 3 is the fp32-faithful mode: operands are (hi, lo) 16-bit planes and each k-step issues
//     hi*hi + hi*lo + lo*hi (the lo*lo term, 2^-22 relative with fp16 planes, is dropped).
#include <stdlib.h>

#include "gdrn_internal.h"
#include "gemm_epilogue.cuh"
#include "gemm_params.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace gdrn {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kSmemBudget = 227 * 1024;
constexpr int kAuxBytes = 4096;  // barriers + [2][BLOCK_N] BatchNorm partial sums
constexpr int kThreads = 288;    // two MMA warpgroups + one producer warp

// BLOCK_M = 256 (gemm_fwd_tall_kernel): every MMA warpgroup owns 128 rows as two 64-row halves, and the A tile is two
// 128-row TMA boxes.  A single-pass k-block then moves 48 KB of operands for 4.2 MFLOP (85 FLOP per byte) instead of 32 KB for
// 2.1 MFLOP (64 FLOP per byte): the single-pass 128 x 128 tile is bound by the L2 -> SM operand traffic, not by the MMAs.
template <int BLOCK_N, int NSPLIT, int BLOCK_M = kBlockM>
struct GemmCfg {
    static constexpr int NPL = (NSPLIT == 1) ? 1 : 2;
    static constexpr int MH = BLOCK_M / kBlockM;  // 64-row MMA halves per warpgroup and 128-row A boxes per stage
    static constexpr int A_BYTES = BLOCK_M * kBlockK * 2;
    static constexpr int B_BYTES = BLOCK_N * kBlockK * 2;
    static constexpr int STAGE_BYTES = NPL * (A_BYTES + B_BYTES);
    static constexpr int STAGES_RAW = (kSmemBudget - kAuxBytes - 1024) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + kAuxBytes + 1024;
    // gemm_fwd_tma_kernel: a 32 KB output staging buffer behind the ring (16 KB per MMA warpgroup: its 64 rows of one 128-wide or
    // two 64-wide 16-bit planes), paid for by a smaller aux area (barriers at +0, the [2][BLOCK_N] partial sums at +512); the ring
    // keeps its stages.  The 256-row tile has 4 stages of 48 KB: 192 KB + 32 KB + 3 KB = 227 KB.
    static constexpr int OUT_STAGE_BYTES = 32768;
    static constexpr int SMEM_BYTES_TMA = STAGES * STAGE_BYTES + OUT_STAGE_BYTES + 2048 + 1024;
    static_assert(SMEM_BYTES_TMA <= kSmemBudget, "no room for the output staging buffer");
    static_assert(512 + 2 * BLOCK_N * 4 <= 2048 && 2 * STAGES * 8 <= 512, "aux area of gemm_fwd_tma_kernel");
    // 3-pass mode: the small cross terms (hi*lo + lo*hi) are kept in their own accumulator and added to the main one with a
    // round-to-nearest fp32 fma before the epilogue.  Each k-step issues three MMAs of width BLOCK_N, each writing one WHOLE
    // accumulator: a_hi x [w_hi; w_lo] as one 2 * BLOCK_N-wide MMA followed by a_lo x w_hi into its upper half would read
    // a_hi once less, but an MMA that writes part of the registers of one still in flight makes ptxas serialise the whole
    // wgmma chain (warning C7511); the three-MMA form measured 0.9 % faster per step.
    static constexpr int NACC = (NSPLIT == 3) ? 2 : 1;
    static constexpr int ACC_REGS = NACC * BLOCK_N / 2;  // per thread and 64-row half: 64 rows x NACC * BLOCK_N columns / 128 threads
    static_assert(STAGES >= 2, "pipeline too shallow");
    static_assert(MH == 1 || (MH == 2 && NSPLIT == 1), "256-row tiles are single-pass only (128 accumulator registers)");
};

// Weight group of an M-tile (GROUPED): tiles never straddle a group (the entry points require rows_per_group % 128 == 0), and
// the group id read from device memory is clamped so that neither the weight tile nor the bias is read outside the tables.
__device__ __forceinline__ int tile_group(const GemmParams& p, int m_tile) {
    const int g = __ldg(p.group + (m_tile * kBlockM) / p.rows_per_group);
    return min(max(g, 0), p.num_w_groups - 1);
}

// BLOCK_M = 256 only with OUT_TMA and a plain epilogue (pick_block_m): bias and activation, one 16-bit output plane; no residual,
// fp32 output, BatchNorm statistics or output-parity phases, so the tall kernel does not carry their code.
template <int BLOCK_N, int NSPLIT, bool GROUPED, bool OUT_TMA, int BLOCK_M = kBlockM>
__device__ __forceinline__ void gemm_fwd_body(const GemmParams& p) {
    using Cfg = GemmCfg<BLOCK_N, NSPLIT, BLOCK_M>;
    constexpr int NPL = Cfg::NPL;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int MH = Cfg::MH;
    constexpr bool PLAIN = MH == 2;
    static_assert(!PLAIN || (OUT_TMA && !GROUPED), "the 256-row tile stores with TMA");
    constexpr int BOX_BYTES = kBlockM * kBlockK * 2;  // one 128-row A box

    // 1024-byte alignment by POINTER arithmetic on the __shared__ array (not through uintptr_t): the compiler keeps the
    // shared address space, so the epilogue's statistics compile to shared-memory atomics instead of generic ones
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* aux = smem + STAGES * Cfg::STAGE_BYTES + (OUT_TMA ? Cfg::OUT_STAGE_BYTES : 0);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty_bar = full_bar + STAGES;
    float* s_stats = reinterpret_cast<float*>(aux + 512);  // [2][BLOCK_N]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;
    const int num_tiles = p.num_m_tiles * p.num_n_tiles;

    if (threadIdx.x == 0) {
        for (int pl = 0; pl < NPL; ++pl) {
            tma_prefetch_desc(&p.tmB[pl]);
            tma_prefetch_desc(&p.tmA[pl][0]);
            if constexpr (OUT_TMA) tma_prefetch_desc(&p.tmC[pl]);
        }
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);  // one arrival per MMA warpgroup
        }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < 2 * BLOCK_N; i += blockDim.x) s_stats[i] = 0.f;
    __syncthreads();
    pdl_launch_dependents();  // the next kernel of the stream may start its prologue under our tail
    pdl_wait();               // nothing above touched global memory; from here on we read what the predecessor wrote
    // persistent CTAs stride over the tile list (phase-major for the stride-2 dgrad)
    const int my_cta = blockIdx.x, num_ctas = gridDim.x;
    const int num_groups = (p.nphase ? p.nphase : 1) * num_tiles;

    if (wg == 2) {
        // ------------------------------------------------------------------ TMA producer
        // Executed by the whole warp with warp-uniform control flow; one elected lane issues.  Taps and channel chunks are
        // nested loops with incremental state: per k-block only the barrier wait, the expect_tx and the TMA issues remain.
        const uint32_t smem_base = smem_u32(smem), full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);
        const uint64_t tmB0 = reinterpret_cast<uint64_t>(&p.tmB[0]), tmB1 = reinterpret_cast<uint64_t>(&p.tmB[1]);
        const int cch = p.cchunks, mode = p.mode, KWv = p.KW, padv = p.pad, stride2 = (p.stride == 2), nph = p.nphase;
        const int ntap_all = mode == 1 ? p.num_kb / (cch > 0 ? cch : 1) : 0;
        int stage = 0;
        uint32_t phase = 0;
        for (int grp = my_cta; grp < num_groups; grp += num_ctas) {
            int rem = grp, tap_base = 0, ntap = ntap_all;
            if (nph) {
                const int ph = grp / num_tiles;
                rem = grp - ph * num_tiles;
                tap_base = p.ph_tap0[ph];
                ntap = p.ph_tap0[ph + 1] - tap_base;
            }
            const int n_tile = rem % p.num_n_tiles;
            const int m_tile = rem / p.num_n_tiles;
            const int bn0 = n_tile * BLOCK_N + (GROUPED ? tile_group(p, m_tile) * p.w_group_rows : 0);
            if (mode == 1) {
                int n0[MH], h0[MH];  // image and first output row of each 128-row box of the tile
#pragma unroll
                for (int b = 0; b < MH; ++b) {
                    const int t = m_tile * MH + b;
                    if (p.TN == 1) {
                        n0[b] = t / p.tiles_per_img;
                        h0[b] = (t - n0[b] * p.tiles_per_img) * p.TH;
                    } else {
                        n0[b] = t * p.TN;
                        h0[b] = 0;
                    }
                }
                int r = 0, s2 = 0;
                for (int t = 0; t < ntap; ++t) {
                    int dh, dw, map = 0, wt = t;
                    if (nph) {
                        dh = p.tap_dh[tap_base + t];
                        dw = p.tap_dw[tap_base + t];
                        wt = p.tap_w[tap_base + t];
                    } else {
                        dh = r - padv;
                        dw = s2 - padv;
                        if (stride2) {
                            map = ((dh & 1) << 1) | (dw & 1);
                            dh >>= 1;  // arithmetic shift == floor division
                            dw >>= 1;
                        }
                        if (++s2 == KWv) {
                            s2 = 0;
                            ++r;
                        }
                    }
                    const uint64_t tmA0 = reinterpret_cast<uint64_t>(&p.tmA[0][map]);
                    const uint64_t tmA1 = reinterpret_cast<uint64_t>(&p.tmA[1][map]);
                    int kw = wt * cch * kBlockK;
                    for (int cc = 0; cc < cch; ++cc, kw += kBlockK) {
                        const uint32_t fb = full0 + stage * 8, dst = smem_base + stage * Cfg::STAGE_BYTES;
                        mbar_wait_u32(empty0 + stage * 8, phase ^ 1);
                        if (elect_one()) {
                            mbar_arrive_expect_tx_u32(fb, Cfg::STAGE_BYTES);
#pragma unroll
                            for (int b = 0; b < MH; ++b) {
                                tma_load_4d_u32(dst + b * BOX_BYTES, tmA0, fb, cc * kBlockK, dw, h0[b] + dh, n0[b]);
                                if (NPL == 2) tma_load_4d_u32(dst + Cfg::A_BYTES + b * BOX_BYTES, tmA1, fb, cc * kBlockK, dw, h0[b] + dh, n0[b]);
                            }
                            tma_load_2d_u32(dst + NPL * Cfg::A_BYTES, tmB0, fb, kw, bn0);
                            if (NPL == 2) tma_load_2d_u32(dst + NPL * Cfg::A_BYTES + Cfg::B_BYTES, tmB1, fb, kw, bn0);
                        }
                        __syncwarp();
                        if (++stage == STAGES) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
            } else {
                const uint64_t tmA0 = reinterpret_cast<uint64_t>(&p.tmA[0][0]);
                const uint64_t tmA1 = reinterpret_cast<uint64_t>(&p.tmA[1][0]);
                const int row0 = m_tile * BLOCK_M;
                for (int kb = 0, kc = 0; kb < p.num_kb; ++kb, kc += kBlockK) {
                    const uint32_t fb = full0 + stage * 8, dst = smem_base + stage * Cfg::STAGE_BYTES;
                    mbar_wait_u32(empty0 + stage * 8, phase ^ 1);
                    if (elect_one()) {
                        mbar_arrive_expect_tx_u32(fb, Cfg::STAGE_BYTES);
#pragma unroll
                        for (int b = 0; b < MH; ++b) {
                            tma_load_2d_u32(dst + b * BOX_BYTES, tmA0, fb, kc, row0 + b * kBlockM);
                            if (NPL == 2) tma_load_2d_u32(dst + Cfg::A_BYTES + b * BOX_BYTES, tmA1, fb, kc, row0 + b * kBlockM);
                        }
                        tma_load_2d_u32(dst + NPL * Cfg::A_BYTES, tmB0, fb, kc, bn0);
                        if (NPL == 2) tma_load_2d_u32(dst + NPL * Cfg::A_BYTES + Cfg::B_BYTES, tmB1, fb, kc, bn0);
                    }
                    __syncwarp();
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- MMA + epilogue warpgroups
    const int cw = wg;  // rows [64 cw, 64 cw + 64) of every tile; of a 256-row tile rows [128 cw, 128 cw + 128)
    const uint64_t desc_const = make_wgmma_desc(0, 16, 1024);
    const uint32_t smem_base = smem_u32(smem), full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);
    const bool signaller = (threadIdx.x & 127) == 0;
    const int cch = p.cchunks, nph = p.nphase, nkb_all = p.num_kb;
    int stage = 0;
    uint32_t phase = 0;
    // TMA-stored output: each warpgroup stages its 64 rows of the 16-bit planes in its own 16 KB half of the staging buffer
    // ([plane][64-column box][64 rows][128 B]) and one thread stores them with TMA while the warpgroup goes on to the next tile's
    // MMAs; the buffer is rewritten only after those stores have read it, normally a whole tile later.  The two planes of a
    // 128-wide 3-pass tile (32 KB) are staged in two 64-column halves, the second once the first half's stores have read the buffer.
    constexpr int PASSES = (BLOCK_N == 128 && NSPLIT == 3) ? 2 : 1;
    constexpr int JP = BLOCK_N / 8 / PASSES;  // column groups per pass
    static_assert(JP * 1024 * NPL <= Cfg::OUT_STAGE_BYTES / 2, "staging buffer too small");
    uint8_t* const stg = smem + STAGES * Cfg::STAGE_BYTES + cw * (Cfg::OUT_STAGE_BYTES / 2);
    auto wg_sync = [&]() {
        if (cw == 0) named_bar_sync<3, 128>();
        else named_bar_sync<4, 128>();
    };
    for (int grp = my_cta; grp < num_groups; grp += num_ctas) {
        int rem = grp, ph = 0, nkb = nkb_all;
        if (nph) {
            ph = grp / num_tiles;
            rem = grp - ph * num_tiles;
            nkb = (p.ph_tap0[ph + 1] - p.ph_tap0[ph]) * cch;
        }
        const int n_tile = rem % p.num_n_tiles;
        const int m_tile = rem / p.num_n_tiles;
        float acc[MH * Cfg::ACC_REGS];  // [64-row half][ACC_REGS]
        int prev_stage = -1;
        for (int kb = 0; kb < nkb; ++kb) {
            const uint32_t a_addr = smem_base + stage * Cfg::STAGE_BYTES;
            const uint64_t da = desc_const | (uint64_t)((a_addr + cw * MH * (64 * 128)) >> 4);
            const uint64_t db = desc_const | (uint64_t)((a_addr + NPL * Cfg::A_BYTES) >> 4);
            mbar_wait_u32(full0 + stage * 8, phase);
            wgmma_fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k) {
                const uint32_t ac = (kb > 0 || k > 0) ? 1u : 0u;
                if constexpr (NSPLIT == 3) {
                    Wgmma<BLOCK_N, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, ac);  // a_hi x w_hi -> main
                    Wgmma<BLOCK_N, 0, 0>::mma(acc + BLOCK_N / 2, da + 2 * k, db + (Cfg::B_BYTES >> 4) + 2 * k, ac);  // a_hi x w_lo -> cross
                    Wgmma<BLOCK_N, 0, 0>::mma(acc + BLOCK_N / 2, da + (Cfg::A_BYTES >> 4) + 2 * k, db + 2 * k, 1u);  // a_lo x w_hi -> cross
                } else {
#pragma unroll
                    for (int h = 0; h < MH; ++h)  // 64-row half h: A rows 64 h further on, (64 * 128) >> 4 descriptor units
                        Wgmma<BLOCK_N, 0, 0>::mma(acc + h * Cfg::ACC_REGS, da + h * 512 + 2 * k, db + 2 * k, ac);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage may be refilled
            wgmma_fence_regs(acc);
            if (prev_stage >= 0 && signaller) mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = stage;
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (prev_stage >= 0 && signaller) mbar_arrive(&empty_bar[prev_stage]);
        if constexpr (NSPLIT == 3) {
            // fold the cross terms into the main accumulator before the epilogue; the empty asm pins each sum here, so the
            // cross registers are dead before the epilogue's address and output work starts
#pragma unroll
            for (int i = 0; i < BLOCK_N / 2; ++i) {
                acc[i] = fmaf(acc[BLOCK_N / 2 + i], kLoInvScale, acc[i]);
                asm volatile("" : "+f"(acc[i]));
            }
        }
        const int row0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);
        if constexpr (GROUPED) {
            gemm_epilogue_tile<BLOCK_N, true>(p, acc, lane, row0, m_tile, n_tile, ph, s_stats, tile_group(p, m_tile) * p.bias_stride);
        } else if constexpr (OUT_TMA) {
            // the 128-row tile holding this warpgroup's rows, and the row of it in acc[4j + 0..1] of the first 64-row half
            const int m128 = MH == 2 ? 2 * m_tile + cw : m_tile;
            const int r0 = MH == 2 ? row0 - cw * 64 : row0;
            const int grow0 = m128 * kBlockM + r0 - (r0 & 63);  // first output row of this warpgroup('s first half)
            auto store = [&](int first_row, int box0) {       // one thread: the staged boxes of both planes
                if (first_row < p.M) {
                    for (int pl = 0; pl < (p.out_lo != nullptr ? 2 : 1); ++pl)
                        for (int b = 0; b < JP / 8; ++b)
                            if (n_tile * BLOCK_N + 64 * (box0 + b) < p.N)
                                tma_store_2d_u32(reinterpret_cast<uint64_t>(&p.tmC[pl]), smem_u32(stg) + (pl * (JP / 8) + b) * 8192,
                                                 n_tile * BLOCK_N + 64 * (box0 + b), first_row);
                }
                bulk_commit_group();
            };
            if (signaller) bulk_wait_group_read<0>();  // the previous stores have read the buffer
            wg_sync();
            gemm_epilogue_tile<BLOCK_N, false, true, 0, JP, PLAIN>(p, acc, lane, r0, m128, n_tile, ph, s_stats, 0, stg);
            fence_proxy_async();  // this thread's st.shared -> visible to the TMA store (async proxy)
            wg_sync();
            if (signaller) store(grow0, 0);
            if constexpr (PASSES == 2) {
                if (signaller) bulk_wait_group_read<0>();
                wg_sync();
                gemm_epilogue_tile<BLOCK_N, false, true, JP, 2 * JP>(p, acc, lane, row0, m_tile, n_tile, ph, s_stats, 0, stg);
                fence_proxy_async();
                wg_sync();
                if (signaller) store(grow0, JP / 8);
            }
            if constexpr (MH == 2) {  // the second 64-row half, once the first half's stores have read the buffer
                if (signaller) bulk_wait_group_read<0>();
                wg_sync();
                gemm_epilogue_tile<BLOCK_N, false, true, 0, JP, PLAIN>(p, acc + Cfg::ACC_REGS, lane, r0 + 64, m128, n_tile, ph, s_stats, 0,
                                                                         stg);
                fence_proxy_async();
                wg_sync();
                if (signaller) store(grow0 + 64, 0);
            }
        } else {
            gemm_epilogue_tile<BLOCK_N>(p, acc, lane, row0, m_tile, n_tile, ph, s_stats);
        }
    }
    if (OUT_TMA && signaller) bulk_wait_group<0>();  // the output is written before the CTA exits
    if (!PLAIN && p.stats != nullptr) {
        asm volatile("bar.sync 1, 256;" ::: "memory");  // the two MMA warpgroups only
        const int n_tile = my_cta % p.num_n_tiles;      // fixed per CTA (num_ctas % num_n_tiles == 0)
        for (int i = threadIdx.x; i < BLOCK_N; i += 256) {
            const int col = n_tile * BLOCK_N + i;
            if (col < p.N) {
                if (p.stats_f64) {
                    atomicAdd(reinterpret_cast<double*>(p.stats) + col, (double)s_stats[i]);
                    atomicAdd(reinterpret_cast<double*>(p.stats) + p.N + col, (double)s_stats[BLOCK_N + i]);
                } else {
                    atomicAdd(p.stats + col, s_stats[i]);
                    atomicAdd(p.stats + p.N + col, s_stats[BLOCK_N + i]);
                }
            }
        }
    }
}

template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(kThreads, 1) gemm_fwd_kernel(const __grid_constant__ GemmParams p) {
    gemm_fwd_body<BLOCK_N, NSPLIT, false, false>(p);
}

// 16-bit output tiles staged in shared memory and written by TMA stores (GemmParams::out_tma, see make_out_maps).
template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(kThreads, 1) gemm_fwd_tma_kernel(const __grid_constant__ GemmParams p) {
    gemm_fwd_body<BLOCK_N, NSPLIT, false, true>(p);
}

// 256-row tiles of the single-pass launches with a plain epilogue (pick_block_m).
template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(kThreads, 1) gemm_fwd_tall_kernel(const __grid_constant__ GemmParams p) {
    gemm_fwd_body<BLOCK_N, NSPLIT, false, true, 2 * kBlockM>(p);
}

// Per-group weights: the class-aware 1x1 output conv and its dgrad, where every crop (4096 rows) reads its class's weight rows.
template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(kThreads, 1) gemm_fwd_grouped_kernel(const __grid_constant__ GemmParams p) {
    gemm_fwd_body<BLOCK_N, NSPLIT, true, false>(p);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <int BLOCK_N, int NSPLIT, bool GROUPED, int BLOCK_M = kBlockM>
static int launch_gemm(const GemmParams& p, cudaStream_t stream) {
    using Cfg = GemmCfg<BLOCK_N, NSPLIT, BLOCK_M>;
    void (*kern)(const GemmParams);
    if constexpr (BLOCK_M != kBlockM) kern = gemm_fwd_tall_kernel<BLOCK_N, NSPLIT>;
    else kern = GROUPED ? gemm_fwd_grouped_kernel<BLOCK_N, NSPLIT>
                        : (p.out_tma ? gemm_fwd_tma_kernel<BLOCK_N, NSPLIT> : gemm_fwd_kernel<BLOCK_N, NSPLIT>);
    static bool attr_set[2] = {false, false};
    if (!attr_set[p.out_tma]) {
        GDRN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          p.out_tma ? Cfg::SMEM_BYTES_TMA : Cfg::SMEM_BYTES));
        attr_set[p.out_tma] = true;
    }
    const int groups = (p.nphase ? p.nphase : 1) * p.num_m_tiles * p.num_n_tiles;
    int ctas = groups < num_sms() ? groups : num_sms();
    ctas -= ctas % p.num_n_tiles;  // every CTA keeps one n_tile => per-CTA BatchNorm partial sums
    if (ctas <= 0) ctas = p.num_n_tiles;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(ctas);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = p.out_tma ? Cfg::SMEM_BYTES_TMA : Cfg::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    int na = 0;
    if (pdl_enabled()) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    GDRN_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
    count_launch();
    return 0;
}

static thread_local int g_last_variant = 0, g_last_block_m = 0;

// p.num_m_tiles counts tiles of block_m rows
template <bool GROUPED>
static int dispatch_gemm(const GemmParams& p, int block_n, int block_m, int nsplit, cudaStream_t stream) {
    g_last_variant = block_n * 10 + nsplit;
    g_last_block_m = block_m;
    if (block_m != kBlockM) {
        if (!GROUPED && block_m == 2 * kBlockM && block_n == 128 && nsplit == 1) return launch_gemm<128, 1, false, 2 * kBlockM>(p, stream);
        return set_error(GDRN_ERR_ARG, "gemm: no %d-row tile for block_n=%d nsplit=%d", block_m, block_n, nsplit);
    }
    if (nsplit == 1) {
        if (block_n == 128) return launch_gemm<128, 1, GROUPED>(p, stream);
        if (block_n == 64) return launch_gemm<64, 1, GROUPED>(p, stream);
    } else if (nsplit == 3) {
        if (block_n == 128) return launch_gemm<128, 3, GROUPED>(p, stream);
        if (block_n == 64) return launch_gemm<64, 3, GROUPED>(p, stream);
    }
    return set_error(GDRN_ERR_ARG, "gemm: unsupported block_n=%d nsplit=%d", block_n, nsplit);
}

static int dispatch_gemm(const GemmParams& p, int block_n, int block_m, int nsplit, cudaStream_t stream) {
    return p.group != nullptr ? dispatch_gemm<true>(p, block_n, block_m, nsplit, stream)
                              : dispatch_gemm<false>(p, block_n, block_m, nsplit, stream);
}

// Grouped weights (gdrn_conv_fwd_grouped / gdrn_gemm_fwd_grouped): the argument checks shared by both, without touching the device.
static int check_groups(const char* fn, const int* group, int M, int rows_per_group, int num_groups, int bias_stride, bool has_bias) {
    if (group == nullptr) return set_error(GDRN_ERR_ARG, "%s: group is NULL", fn);
    if (num_groups < 1) return set_error(GDRN_ERR_ARG, "%s: num_groups=%d must be >= 1", fn, num_groups);
    if (rows_per_group <= 0 || rows_per_group % kBlockM != 0)
        return set_error(GDRN_ERR_ARG, "%s: rows_per_group=%d must be a positive multiple of %d (tiles never straddle a group)", fn,
                         rows_per_group, kBlockM);
    if (M % rows_per_group != 0) return set_error(GDRN_ERR_ARG, "%s: M=%d is not a whole number of groups of %d rows", fn, M, rows_per_group);
    if (has_bias && bias_stride < 0) return set_error(GDRN_ERR_ARG, "%s: bias_stride=%d must be >= 0", fn, bias_stride);
    return 0;
}

// Launches whose 16-bit planes leave through TMA stores (gemm_fwd_tma_kernel): every mode 0 / mode 1 launch with a 16-bit output.
// Phase-decomposed dgrads (which scatter their rows) and the grouped kernel store directly, and so does a single-pass launch
// that writes two planes (only one 128-wide plane fits a warpgroup's half of the staging buffer).
// The output map is [M][min(ldc, N rounded up to 32)]: rows beyond M and the 32-column chunks that start at or beyond N are not
// written, the columns [N, ldc) of a partial chunk are written as zeros, exactly like the direct stores.
static int make_out_maps(GemmParams& p, int nsplit) {
    if (p.out_hi == nullptr || p.group != nullptr || (p.out_lo != nullptr && nsplit == 1)) return 0;
    const int width = p.ldc < (p.N + 31) / 32 * 32 ? p.ldc : (p.N + 31) / 32 * 32;
    uint64_t dims[2] = {(uint64_t)width, (uint64_t)p.M};
    uint64_t strides[1] = {(uint64_t)p.ldc * 2};
    uint32_t box[2] = {64, 64};
    if (make_tmap(&p.tmC[0], p.out_hi, 2, dims, strides, box)) return GDRN_ERR_CUDA;
    if (p.out_lo != nullptr && make_tmap(&p.tmC[1], p.out_lo, 2, dims, strides, box)) return GDRN_ERR_CUDA;
    p.out_tma = 1;
    return 0;
}

// Tile width: the widest BLOCK_N (fewest A re-reads, best smem-bandwidth ratio) that still yields >= ~0.75 waves of
// CTAs on the SMs; small-M layers (layer4, FC) fall back to narrower tiles instead of leaving SMs idle.
static int pick_block_n(int n_pad, int num_m_tiles) {
    if (n_pad % 64 != 0) return -1;
    if (n_pad % 128 == 0 && num_m_tiles * (n_pad / 128) >= (num_sms() * 3) / 4) return 128;
    if (num_m_tiles * (n_pad / 128) < num_sms() / 2) return 64;
    return n_pad % 128 == 0 ? 128 : 64;
}

// Tile height, after pick_block_n has fixed the width from the 128-row tile count: 256 rows (gemm_fwd_tall_kernel) for a
// single-pass 128-wide launch whose epilogue is plain -- a TMA-stored 16-bit plane (make_out_maps; so not grouped), no lo plane,
// residual, fp32 output, BatchNorm statistics or output-parity phases -- while the 256-row tiles still fill >= ~0.75 waves.
static int pick_block_m(const GemmParams& p, int block_n, int nsplit) {
    const bool plain = p.out_tma && p.out_lo == nullptr && p.res_hi == nullptr && p.out_f32 == nullptr && p.stats == nullptr &&
                       p.group == nullptr && p.nphase == 0;
    const int tall_tiles = (p.M + 2 * kBlockM - 1) / (2 * kBlockM) * p.num_n_tiles;
    return nsplit == 1 && block_n == 128 && plain && tall_tiles >= (num_sms() * 3) / 4 ? 2 * kBlockM : kBlockM;
}

// Sets the tile height and the M-tile count of a launch whose GemmParams are otherwise complete.
static int set_block_m(GemmParams& p, int block_n, int nsplit) {
    const int block_m = pick_block_m(p, block_n, nsplit);
    p.num_m_tiles = (p.M + block_m - 1) / block_m;
    return block_m;
}

}  // namespace gdrn

using namespace gdrn;

static int conv_fwd_impl(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                         float* y_f32, const float* bias, const void* res_hi, const void* res_lo, float* stats, int N, int H, int W,
                         int Cin, int Cout, int Cout_pad, int KH, int KW, int stride, int pad, int ldc, int act, int nsplit,
                         const int* group, int rows_per_group, int num_groups, int bias_stride, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (nsplit != 1 && nsplit != 3) return set_error(GDRN_ERR_ARG, "conv_fwd: nsplit must be 1 or 3");
    if (nsplit == 3 && (x_lo == nullptr || w_lo == nullptr)) return set_error(GDRN_ERR_ARG, "conv_fwd: lo planes missing");
    if (Cin % 64 != 0) return set_error(GDRN_ERR_ARG, "conv_fwd: Cin=%d must be a multiple of 64", Cin);
    if (stride != 1 && stride != 2) return set_error(GDRN_ERR_ARG, "conv_fwd: stride must be 1 or 2");
    if (H % stride || W % stride) return set_error(GDRN_ERR_ARG, "conv_fwd: H, W must be divisible by stride");
    if (ldc % 8 != 0 || ldc < Cout) return set_error(GDRN_ERR_ARG, "conv_fwd: bad ldc=%d", ldc);
    if (res_hi != nullptr && (Cout % 32 != 0 || y_hi == nullptr))
        return set_error(GDRN_ERR_ARG, "conv_fwd: a residual needs Cout %% 32 == 0 and a 16-bit output");
    if ((act & ~kActStatsF64) < 0 || (act & ~kActStatsF64) > 2) return set_error(GDRN_ERR_ARG, "conv_fwd: act must be 0 (none), 1 (LeakyReLU 0.1) or 2 (ReLU)");
    const int Ho = H / stride, Wo = W / stride;
    if (Wo > 128 || 128 % Wo != 0) return set_error(GDRN_ERR_ARG, "conv_fwd: unsupported output width %d", Wo);
    if ((uint64_t)N * Ho * Wo * ldc > UINT32_MAX) return set_error(GDRN_ERR_ARG, "conv_fwd: output too large for 32-bit offsets");
    int TH = 128 / Wo;
    if (TH > Ho) TH = Ho;
    const int TN = 128 / (Wo * TH);
    if (Ho % TH != 0) return set_error(GDRN_ERR_ARG, "conv_fwd: Ho=%d not divisible by tile rows %d", Ho, TH);
    const int block_n = pick_block_n(Cout_pad, (N * Ho * Wo + 127) / 128);
    if (block_n < 0) return set_error(GDRN_ERR_ARG, "conv_fwd: Cout_pad=%d must be a multiple of 64", Cout_pad);

    GemmParams p;
    memset(&p, 0, sizeof(p));
    const int npl = nsplit == 1 ? 1 : 2;
    const void* xs[2] = {x_hi, x_lo};
    const void* ws[2] = {w_hi, w_lo};
    const int K = KH * KW * Cin;
    for (int pl = 0; pl < npl; ++pl) {
        const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(xs[pl]);
        for (int ph = 0; ph < (stride == 2 ? 4 : 1); ++ph) {
            const int phh = ph >> 1, phw = ph & 1;
            uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)N};
            uint64_t strides[3] = {(uint64_t)stride * Cin * 2, (uint64_t)stride * W * Cin * 2, (uint64_t)H * W * Cin * 2};
            uint32_t box[4] = {64, (uint32_t)Wo, (uint32_t)TH, (uint32_t)TN};
            const void* base = xb + ((size_t)phh * W + phw) * Cin;
            if (make_tmap(&p.tmA[pl][ph], base, 4, dims, strides, box)) return GDRN_ERR_CUDA;
        }
        uint64_t wdims[2] = {(uint64_t)K, (uint64_t)Cout_pad * num_groups};
        uint64_t wstr[1] = {(uint64_t)K * 2};
        uint32_t wbox[2] = {64, (uint32_t)block_n};
        if (make_tmap(&p.tmB[pl], ws[pl], 2, wdims, wstr, wbox)) return GDRN_ERR_CUDA;
    }
    p.mode = 1;
    p.M = N * Ho * Wo;
    p.N = Cout;
    p.num_m_tiles = (p.M + 127) / 128;
    p.num_n_tiles = Cout_pad / block_n;
    p.cchunks = Cin / 64;
    p.num_kb = KH * KW * p.cchunks;
    p.KW = KW;
    p.pad = pad;
    p.stride = stride;
    p.TH = TH;
    p.TN = TN;
    p.tiles_per_img = (TN == 1) ? Ho / TH : 0;
    p.out_hi = y_hi;
    p.out_lo = y_lo;
    p.out_f32 = y_f32;
    p.ldc = ldc;
    p.bias = bias;
    p.res_hi = res_hi;
    p.res_lo = res_lo;
    p.act = act & ~kActStatsF64;
    p.stats = stats;
    p.stats_f64 = (act & kActStatsF64) ? 1 : 0;
    p.group = group;
    p.rows_per_group = rows_per_group;
    p.w_group_rows = Cout_pad;
    p.num_w_groups = num_groups;
    p.bias_stride = bias_stride;
    if (make_out_maps(p, nsplit)) return GDRN_ERR_CUDA;
    return dispatch_gemm(p, block_n, set_block_m(p, block_n, nsplit), nsplit, stream);
}

extern "C" int gdrn_conv_fwd(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, void* y_hi,
                             void* y_lo, float* y_f32, const float* bias, const void* res_hi, const void* res_lo, float* stats,
                             int N, int H, int W, int Cin, int Cout, int Cout_pad, int KH, int KW, int stride, int pad, int ldc,
                             int act, int nsplit, void* stream_) {
    return conv_fwd_impl(x_hi, x_lo, w_hi, w_lo, y_hi, y_lo, y_f32, bias, res_hi, res_lo, stats, N, H, W, Cin, Cout, Cout_pad, KH,
                         KW, stride, pad, ldc, act, nsplit, nullptr, 0, 1, 0, stream_);
}

// Class-aware 1x1 output conv: w holds num_groups weight blocks of Cout_pad rows ([num_groups * Cout_pad][K]), bias num_groups
// blocks of bias_stride floats; output rows [g * rows_per_group, (g + 1) * rows_per_group) use block group[g] (a device array of
// M / rows_per_group ints, clamped to [0, num_groups)).  No residual and no BatchNorm statistics.
extern "C" int gdrn_conv_fwd_grouped(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                                     float* y_f32, const float* bias, int N, int H, int W, int Cin, int Cout, int Cout_pad, int KH,
                                     int KW, int stride, int pad, int ldc, int act, int nsplit, const int* group, int rows_per_group,
                                     int num_groups, int bias_stride, void* stream_) {
    const int M = N * (H / (stride > 0 ? stride : 1)) * (W / (stride > 0 ? stride : 1));
    if (int rc = check_groups("conv_fwd_grouped", group, M, rows_per_group, num_groups, bias_stride, bias != nullptr)) return rc;
    if (act & kActStatsF64) return set_error(GDRN_ERR_ARG, "conv_fwd_grouped: no BatchNorm statistics");
    return conv_fwd_impl(x_hi, x_lo, w_hi, w_lo, y_hi, y_lo, y_f32, bias, nullptr, nullptr, nullptr, N, H, W, Cin, Cout, Cout_pad, KH,
                         KW, stride, pad, ldc, act, nsplit, group, rows_per_group, num_groups, bias_stride, stream_);
}

// Data gradient of a stride-2 convolution (k = 3, pad 1; k = 1, pad 0; k = 4, pad 1; k = 2, pad 0), decomposed by OUTPUT
// PARITY: the pixels (2i + a, 2j + b) of dX only receive the filter taps r = a + pad (mod 2), so each of the four phases is a
// small stride-1 conv over the UN-dilated dY -- k = 3: 1 / 2 / 2 / 4 taps, 9 taps per 4 output pixels instead of the 36 of the
// "conv over zero-inserted dY" formulation; k = 4: 2x2 taps per phase; k = 2: one tap per phase -- and no zero-inserted tensor
// in HBM.  One launch covers all phases.
//   du [N][Ho][Wo][Cy] (Cy % 64 == 0), w = the dgrad-packed weights [Cx_pad][K*K*Cy] with flipped taps (pack_conv_dgrad),
//   dx [N][2Ho][2Wo][ldc].  k = 1: only phase (0, 0) is computed, the caller passes a zero-filled dx.
extern "C" int gdrn_conv_dgrad_s2(const void* du_hi, const void* du_lo, const void* w_hi, const void* w_lo, void* dx_hi,
                                  void* dx_lo, const float* bias, float* stats, int N, int Ho, int Wo, int Cy, int Cx, int Cx_pad,
                                  int K, int pad, int ldc, int act, int nsplit, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (nsplit != 1 && nsplit != 3) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: nsplit must be 1 or 3");
    if (nsplit == 3 && (du_lo == nullptr || w_lo == nullptr)) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: lo planes missing");
    if (!((K == 3 && pad == 1) || (K == 1 && pad == 0) || (K == 4 && pad == 1) || (K == 2 && pad == 0)))
        return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: k3 p1, k1 p0, k4 p1 or k2 p0 only (got k%d p%d)", K, pad);
    if (Cy % 64 != 0) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: Cy=%d must be a multiple of 64", Cy);
    if (ldc % 8 != 0 || ldc < Cx) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: bad ldc=%d", ldc);
    if (Wo > 128 || 128 % Wo != 0 || (Ho & (Ho - 1)) != 0) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: unsupported dY size %dx%d", Ho, Wo);
    if ((uint64_t)N * 4 * Ho * Wo * ldc > UINT32_MAX) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: output too large for 32-bit offsets");
    int TH = 128 / Wo;
    if (TH > Ho) TH = Ho;
    const int TN = 128 / (Wo * TH);
    if (Ho % TH != 0) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: Ho=%d not divisible by tile rows %d", Ho, TH);
    const int num_m_tiles = (N * Ho * Wo + 127) / 128;
    const int nphase = K == 1 ? 1 : 4;
    const int block_n = pick_block_n(Cx_pad, num_m_tiles * nphase);
    if (block_n < 0) return set_error(GDRN_ERR_ARG, "conv_dgrad_s2: Cx_pad=%d must be a multiple of 64", Cx_pad);

    GemmParams p;
    memset(&p, 0, sizeof(p));
    const int npl = nsplit == 1 ? 1 : 2;
    const void* xs[2] = {du_hi, du_lo};
    const void* ws[2] = {w_hi, w_lo};
    const int Kw = K * K * Cy;
    for (int pl = 0; pl < npl; ++pl) {
        uint64_t dims[4] = {(uint64_t)Cy, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)N};
        uint64_t strides[3] = {(uint64_t)Cy * 2, (uint64_t)Wo * Cy * 2, (uint64_t)Ho * Wo * Cy * 2};
        uint32_t box[4] = {64, (uint32_t)Wo, (uint32_t)TH, (uint32_t)TN};
        if (make_tmap(&p.tmA[pl][0], xs[pl], 4, dims, strides, box)) return GDRN_ERR_CUDA;
        uint64_t wdims[2] = {(uint64_t)Kw, (uint64_t)Cx_pad};
        uint64_t wstr[1] = {(uint64_t)Kw * 2};
        uint32_t wbox[2] = {64, (uint32_t)block_n};
        if (make_tmap(&p.tmB[pl], ws[pl], 2, wdims, wstr, wbox)) return GDRN_ERR_CUDA;
    }
    p.mode = 1;
    p.M = N * Ho * Wo;
    p.N = Cx;
    p.num_m_tiles = num_m_tiles;
    p.num_n_tiles = Cx_pad / block_n;
    p.cchunks = Cy / 64;
    p.KW = K;
    p.pad = pad;
    p.stride = 1;
    p.TH = TH;
    p.TN = TN;
    p.tiles_per_img = (TN == 1) ? Ho / TH : 0;
    p.out_hi = dx_hi;
    p.out_lo = dx_lo;
    p.ldc = ldc;
    p.bias = bias;    // the same kernel is the FORWARD of ConvTranspose2d(k3, s2, p1, op1) (cdpn_rot_head_region.py:82-91): then
    p.act = act & ~kActStatsF64;  // bias / activation (folded eval BatchNorm) and the BatchNorm batch statistics apply to its output
    p.stats = stats;
    p.stats_f64 = (act & kActStatsF64) ? 1 : 0;
    // phases in order of decreasing tap count (longest tiles first on the persistent CTAs; k = 4 and k = 2 phases are all equal)
    p.nphase = nphase;
    int nt = 0;
    const int order[4][2] = {{1, 1}, {1, 0}, {0, 1}, {0, 0}};
    for (int q = 0; q < nphase; ++q) {
        const int a = K == 1 ? 0 : order[q][0], b = K == 1 ? 0 : order[q][1];
        p.ph_a[q] = a;
        p.ph_b[q] = b;
        p.ph_tap0[q] = nt;
        for (int r = 0; r < K; ++r) {
            if ((a + pad - r) & 1) continue;
            for (int s2 = 0; s2 < K; ++s2) {
                if ((b + pad - s2) & 1) continue;
                p.tap_dh[nt] = (signed char)((a + pad - r) / 2);
                p.tap_dw[nt] = (signed char)((b + pad - s2) / 2);
                p.tap_w[nt] = (signed char)((K - 1 - r) * K + (K - 1 - s2));  // pack_conv_dgrad stores flipped taps
                ++nt;
            }
        }
    }
    p.ph_tap0[nphase] = nt;  // <= 16 = sizeof(p.tap_dh)
    p.num_kb = nt * p.cchunks;  // bookkeeping only (per-tile counts come from the phase table)
    for (p.pw_log2 = 0; (1 << p.pw_log2) < Wo; ++p.pw_log2) {}
    for (p.ph_log2 = 0; (1 << p.ph_log2) < Ho; ++p.ph_log2) {}
    return dispatch_gemm(p, block_n, kBlockM, nsplit, stream);
}

static int gemm_fwd_impl(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                         float* y_f32, const float* bias, float* stats, int M, int N, int N_pad, int K, int ldc, int act, int nsplit,
                         const int* group, int rows_per_group, int num_groups, int bias_stride, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (nsplit != 1 && nsplit != 3) return set_error(GDRN_ERR_ARG, "gemm_fwd: nsplit must be 1 or 3");
    if (nsplit == 3 && (a_lo == nullptr || w_lo == nullptr)) return set_error(GDRN_ERR_ARG, "gemm_fwd: lo planes missing");
    if (K % 64 != 0) return set_error(GDRN_ERR_ARG, "gemm_fwd: K=%d must be a multiple of 64", K);
    if (ldc % 8 != 0 || ldc < N) return set_error(GDRN_ERR_ARG, "gemm_fwd: bad ldc=%d", ldc);
    if ((uint64_t)M * ldc > UINT32_MAX) return set_error(GDRN_ERR_ARG, "gemm_fwd: output too large for 32-bit offsets");
    const int block_n = pick_block_n(N_pad, (M + 127) / 128);
    if (block_n < 0) return set_error(GDRN_ERR_ARG, "gemm_fwd: N_pad=%d must be a multiple of 64", N_pad);
    GemmParams p;
    memset(&p, 0, sizeof(p));
    const int npl = nsplit == 1 ? 1 : 2;
    const void* as[2] = {a_hi, a_lo};
    const void* ws[2] = {w_hi, w_lo};
    for (int pl = 0; pl < npl; ++pl) {
        uint64_t adims[2] = {(uint64_t)K, (uint64_t)M};
        uint64_t astr[1] = {(uint64_t)K * 2};
        uint32_t abox[2] = {64, 128};
        if (make_tmap(&p.tmA[pl][0], as[pl], 2, adims, astr, abox)) return GDRN_ERR_CUDA;
        uint64_t wdims[2] = {(uint64_t)K, (uint64_t)N_pad * num_groups};
        uint32_t wbox[2] = {64, (uint32_t)block_n};
        if (make_tmap(&p.tmB[pl], ws[pl], 2, wdims, astr, wbox)) return GDRN_ERR_CUDA;
    }
    p.mode = 0;
    p.M = M;
    p.N = N;
    p.num_m_tiles = (M + 127) / 128;
    p.num_n_tiles = N_pad / block_n;
    p.num_kb = K / 64;
    p.out_hi = y_hi;
    p.out_lo = y_lo;
    p.out_f32 = y_f32;
    p.ldc = ldc;
    p.bias = bias;
    p.act = act & ~kActStatsF64;
    p.stats = stats;
    p.stats_f64 = (act & kActStatsF64) ? 1 : 0;
    p.group = group;
    p.rows_per_group = rows_per_group;
    p.w_group_rows = N_pad;
    p.num_w_groups = num_groups;
    p.bias_stride = bias_stride;
    if (make_out_maps(p, nsplit)) return GDRN_ERR_CUDA;
    return dispatch_gemm(p, block_n, set_block_m(p, block_n, nsplit), nsplit, stream);
}

extern "C" int gdrn_gemm_fwd(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, void* y_hi,
                             void* y_lo, float* y_f32, const float* bias, float* stats, int M, int N, int N_pad, int K,
                             int ldc, int act, int nsplit, void* stream_) {
    return gemm_fwd_impl(a_hi, a_lo, w_hi, w_lo, y_hi, y_lo, y_f32, bias, stats, M, N, N_pad, K, ldc, act, nsplit, nullptr, 0, 1, 0,
                         stream_);
}

// Grouped plain GEMM (the class-aware output conv's dgrad): w = [num_groups * N_pad][K], rows [g * rows_per_group, ...) of a use
// weight block group[g] (clamped) and bias + group[g] * bias_stride.  No BatchNorm statistics.
extern "C" int gdrn_gemm_fwd_grouped(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                                     float* y_f32, const float* bias, int M, int N, int N_pad, int K, int ldc, int act, int nsplit,
                                     const int* group, int rows_per_group, int num_groups, int bias_stride, void* stream_) {
    if (int rc = check_groups("gemm_fwd_grouped", group, M, rows_per_group, num_groups, bias_stride, bias != nullptr)) return rc;
    if (act & kActStatsF64) return set_error(GDRN_ERR_ARG, "gemm_fwd_grouped: no BatchNorm statistics");
    return gemm_fwd_impl(a_hi, a_lo, w_hi, w_lo, y_hi, y_lo, y_f32, bias, nullptr, M, N, N_pad, K, ldc, act, nsplit, group,
                         rows_per_group, num_groups, bias_stride, stream_);
}

// BLOCK_N * 10 + NSPLIT of the most recent gdrn_conv_fwd / gdrn_gemm_fwd call on this thread
extern "C" int gdrn_last_gemm_variant() { return g_last_variant; }

// tile height (128 or 256 rows) of the same call
extern "C" int gdrn_last_gemm_block_m() { return g_last_block_m; }
