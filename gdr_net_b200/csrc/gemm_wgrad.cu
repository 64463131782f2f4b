// wgmma weight-gradient kernel (sm_90a):  dW[co][tap][ci] = sum_p dY[p][co] * X[p (+) tap][ci]
//
// Both operands are "MN-major" for the tensor core: the reduction index is the pixel p, which is the
// SLOW index of the NHWC tensors, so the 64-pixel x 64-channel TMA boxes land in shared memory as
// [k = pixel][64 channels = 128 B] rows -- exactly the MN-major 128B-swizzled canonical layout
// (wgmma transpose flags set, SBO = 1024 B between 8-pixel groups, LBO = 8192 B between
// 64-channel chunks).  No transposes are ever materialised.
//
//   * A tile = dY  [64 pixels][128 co]      (2 boxes of 64 channels, plain 2-D view [P][Cout])
//   * B tile = X   [64 pixels][<=256 ci]    (<=4 boxes; for a conv the box is the tap-shifted 4-D
//                  window of the NHWC input, zero-filled outside the image; stride-2 convs read the
//                  four parity sub-lattices, like the forward kernel)
//   * one CTA = (co tile, ci tile, tap, K-split); warpgroups 0 and 1 each own 64 output channels (one dY
//     box) with fp32 accumulators in registers, warp 8 is the TMA producer; partial results go to a
//     [ksplit][Cout][taps*Cin] fp32 workspace that the unpack kernel (pack.cu) reduces and transposes
//     into the reference's OIHW gradient layout.
// Backward call sites replaced: autograd wgrad of every nn.Conv2d / ConvTranspose2d / nn.Linear in
// reference resnet_backbone.py, cdpn_rot_head_region.py, conv_pnp_net.py (cuDNN/cuBLAS today).
#include <stdlib.h>

#include "gdrn_internal.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace gdrn {

struct WgradParams {
    CUtensorMap tmA[2];     // dY  [plane]
    CUtensorMap tmB[2][4];  // X   [plane][phase]
    int mode;               // 0 = 2-D GEMM (B = [P][Ntot]), 1 = conv
    int Mvalid;             // Cout
    int Ntot;               // Cin (conv) or total B columns (gemm)
    int num_m_tiles, num_n_tiles, taps, ksplit;
    int kb_total;           // number of 64-pixel blocks
    int KW, pad, stride;
    int blocks_per_img, THk, TNk;
    float* ws;              // [ksplit][num_m_tiles*128][taps*Ntot]
    int tap_pack;           // 1: Cin == 64, stride 1: one work item covers a whole filter ROW, its KW taps packed along N
    int items;              // work items per (m_tile, n_tile, ksplit): taps, or KH when tap_pack
    int ws_ld;              // workspace row length in floats (= KH*KW*Cin)
};

constexpr int kWgStageA = 2 * 8192;
constexpr int kWgThreads = 288;  // warps 0-7: two MMA warpgroups (64 output channels each), warp 8: TMA producer

template <int N_TILE, int NSPLIT>
struct WgradCfg {
    static constexpr int NPL = (NSPLIT == 1) ? 1 : 2;
    static constexpr int NCH = N_TILE / 64;
    static constexpr int A_BYTES = kWgStageA;
    static constexpr int B_BYTES = NCH * 8192;
    static constexpr int STAGE_BYTES = NPL * (A_BYTES + B_BYTES);
    static constexpr int STAGES_RAW = (227 * 1024 - 2048) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2048;
    // 3-pass mode: the cross terms get their own accumulator, added with a round-to-nearest fp32 fma in the epilogue
    static constexpr int NACC = (NSPLIT == 3) ? 2 : 1;
    static constexpr int ACC = N_TILE / 2;  // registers per accumulator set: 64 rows x N_TILE columns over 128 threads
    static_assert(STAGES >= 2, "pipeline too shallow");
};

template <int N_TILE, int NSPLIT>
__global__ void __launch_bounds__(kWgThreads, 1) gemm_wgrad_kernel(const __grid_constant__ WgradParams p) {
    using Cfg = WgradCfg<N_TILE, NSPLIT>;
    constexpr int NPL = Cfg::NPL;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int NCH = Cfg::NCH;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* aux = smem + STAGES * Cfg::STAGE_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // work item decode: m fastest, then n, tap, ksplit
    int item = blockIdx.x;
    const int m_tile = item % p.num_m_tiles;
    item /= p.num_m_tiles;
    const int n_tile = item % p.num_n_tiles;
    item /= p.num_n_tiles;
    const int tap = item % p.items;  // filter tap, or filter row when tap_pack
    const int ks = item / p.items;
    const int kb_per = (p.kb_total + p.ksplit - 1) / p.ksplit;
    const int kb_begin = ks * kb_per;
    const int kb_end = min(p.kb_total, kb_begin + kb_per);
    const int nkb = kb_end - kb_begin;  // may be <= 0 for a ragged last split: then we store zeros

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);  // one arrival per MMA warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();  // the next kernel of the stream may start its prologue under our tail
    pdl_wait();               // nothing above touched global memory; from here on we read what the predecessor wrote

    if (warp == 8) {
        // TMA producer: the whole warp runs the loop (warp-uniform control flow, operands in uniform registers), one elected
        // lane issues; per k-block nothing but the barrier wait, the expect_tx and the issues remains.
        if (nkb > 0) {
            int dh = 0, dw = 0, map = 0;
            if (p.mode == 1 && p.tap_pack) {
                dh = tap - p.pad;  // `tap` is the filter row; the column shift varies per 64-channel chunk below
            } else if (p.mode == 1) {
                const int r = tap / p.KW;
                const int s = tap - r * p.KW;
                dh = r - p.pad;
                dw = s - p.pad;
                if (p.stride == 2) {
                    map = ((dh & 1) << 1) | (dw & 1);
                    dh >>= 1;
                    dw >>= 1;
                }
            }
            const uint32_t smem_base = smem_u32(smem), full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);
            const uint64_t tmA0 = reinterpret_cast<uint64_t>(&p.tmA[0]), tmA1 = reinterpret_cast<uint64_t>(&p.tmA[1]);
            const uint64_t tmB0 = reinterpret_cast<uint64_t>(&p.tmB[0][map]), tmB1 = reinterpret_cast<uint64_t>(&p.tmB[1][map]);
            const int mode = p.mode, tap_pack = p.tap_pack, padv = p.pad, bpi = p.blocks_per_img, THk = p.THk, TNk = p.TNk;
            const int m0 = m_tile * 128, nb0 = n_tile * N_TILE;
            // (image, 64-pixel block inside the image) of the first k-block, advanced incrementally
            int n0 = 0, hb = 0;
            if (mode == 1) {
                if (TNk == 1) {
                    n0 = kb_begin / bpi;
                    hb = kb_begin - n0 * bpi;
                } else {
                    n0 = kb_begin * TNk;
                }
            }
            int stage = 0;
            uint32_t phase = 0;
            for (int kb = kb_begin; kb < kb_end; ++kb) {
                const uint32_t fb = full0 + stage * 8, dst = smem_base + stage * Cfg::STAGE_BYTES;
                const int hh = hb * THk + dh, prow = kb * 64;
                mbar_wait_u32(empty0 + stage * 8, phase ^ 1);
                if (elect_one()) {
                    mbar_arrive_expect_tx_u32(fb, Cfg::STAGE_BYTES);
#pragma unroll
                    for (int pl = 0; pl < NPL; ++pl) {
                        const uint32_t a_dst = dst + pl * Cfg::A_BYTES;
                        const uint64_t tmA = pl ? tmA1 : tmA0, tmB = pl ? tmB1 : tmB0;
                        tma_load_2d_u32(a_dst, tmA, fb, m0, prow);
                        tma_load_2d_u32(a_dst + 8192, tmA, fb, m0 + 64, prow);
                        const uint32_t b_dst = dst + NPL * Cfg::A_BYTES + pl * Cfg::B_BYTES;
                        if (mode == 1) {
                            if (tap_pack) {
#pragma unroll
                                for (int c = 0; c < NCH; ++c)  // chunk c = filter column c (all 64 input channels)
                                    tma_load_4d_u32(b_dst + c * 8192, tmB, fb, 0, c - padv, hh, n0);
                            } else {
#pragma unroll
                                for (int c = 0; c < NCH; ++c)
                                    tma_load_4d_u32(b_dst + c * 8192, tmB, fb, nb0 + c * 64, dw, hh, n0);
                            }
                        } else {
#pragma unroll
                            for (int c = 0; c < NCH; ++c) tma_load_2d_u32(b_dst + c * 8192, tmB, fb, nb0 + c * 64, prow);
                        }
                    }
                }
                __syncwarp();
                if (mode == 1) {
                    if (TNk == 1) {
                        if (++hb == bpi) {
                            hb = 0;
                            ++n0;
                        }
                    } else {
                        n0 += TNk;
                    }
                }
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- MMA + epilogue warpgroups
    const int cw = threadIdx.x >> 7;  // output channels [64 cw, 64 cw + 64) of the tile = dY box cw
    float acc[Cfg::NACC * Cfg::ACC];
    if (nkb > 0) {
        const uint64_t desc_const = make_wgmma_desc(0, 8192, 1024);  // only the 14-bit address field varies
        const uint32_t smem_base = smem_u32(smem), full0 = smem_u32(full_bar);
        const bool signaller = (threadIdx.x & 127) == 0;
        int stage = 0, prev_stage = -1;
        uint32_t phase = 0;
        for (int kb = 0; kb < nkb; ++kb) {
            const uint32_t a_addr = smem_base + stage * Cfg::STAGE_BYTES;
            const uint64_t da = desc_const | (uint64_t)((a_addr + cw * 8192) >> 4);
            const uint64_t db = desc_const | (uint64_t)((a_addr + NPL * Cfg::A_BYTES) >> 4);
            mbar_wait_u32(full0 + stage * 8, phase);
            wgmma_fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {  // 16 pixels (= 16 rows of 128 B = 2048 B) per MMA
                const uint32_t ac = (kb | k) != 0 ? 1u : 0u;
                Wgmma<N_TILE, 1, 1>::mma(acc, da + 128 * k, db + 128 * k, ac);
                if constexpr (NSPLIT == 3) {
                    Wgmma<N_TILE, 1, 1>::mma(acc + Cfg::ACC, da + 128 * k, db + (Cfg::B_BYTES >> 4) + 128 * k, ac);  // hi x lo
                    Wgmma<N_TILE, 1, 1>::mma(acc + Cfg::ACC, da + (Cfg::A_BYTES >> 4) + 128 * k, db + 128 * k, 1u);  // lo x hi
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
    } else {
#pragma unroll
        for (int i = 0; i < Cfg::NACC * Cfg::ACC; ++i) acc[i] = 0.f;
    }
    // fragment layout (wgmma.cuh): acc[4j + 2h + e] = channel row (warp % 4) * 16 + lane / 4 + 8h, column 8j + 2 (lane % 4) + e
    const size_t ld = (size_t)p.ws_ld;
    // tap_pack: columns (filter column, ci) of filter row `tap` are contiguous in the [co][tap][ci] workspace row
    const size_t col0 = p.tap_pack ? (size_t)tap * N_TILE : (size_t)tap * p.Ntot + (size_t)n_tile * N_TILE;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int co = m_tile * 128 + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        float* dst_row = p.ws + ((size_t)ks * p.num_m_tiles * 128 + co) * ld + col0;
#pragma unroll
        for (int j = 0; j < N_TILE / 8; ++j) {
            const int cl = 8 * j + 2 * (lane & 3);
            if (!p.tap_pack && n_tile * N_TILE + cl >= p.Ntot) continue;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                v[e] = acc[4 * j + 2 * h + e];
                if (NSPLIT == 3) v[e] = fmaf(acc[Cfg::ACC + 4 * j + 2 * h + e], kLoInvScale, v[e]);
            }
            *reinterpret_cast<float2*>(dst_row + cl) = make_float2(v[0], v[1]);
        }
    }
}

template <int N_TILE, int NSPLIT>
static int launch_wgrad(const WgradParams& p, cudaStream_t stream) {
    using Cfg = WgradCfg<N_TILE, NSPLIT>;
    auto kern = gemm_wgrad_kernel<N_TILE, NSPLIT>;
    static bool attr_set = false;
    if (!attr_set) {
        GDRN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_set = true;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(p.num_m_tiles * p.num_n_tiles * p.items * p.ksplit);
    cfg.blockDim = dim3(kWgThreads);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
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

static int dispatch_wgrad(const WgradParams& p, int n_tile, int nsplit, cudaStream_t stream) {
    if (nsplit == 1) {
        if (n_tile == 256) return launch_wgrad<256, 1>(p, stream);
        if (n_tile == 192) return launch_wgrad<192, 1>(p, stream);
        if (n_tile == 128) return launch_wgrad<128, 1>(p, stream);
        if (n_tile == 64) return launch_wgrad<64, 1>(p, stream);
    } else if (nsplit == 3) {
        if (n_tile == 128) return launch_wgrad<128, 3>(p, stream);
        if (n_tile == 64) return launch_wgrad<64, 3>(p, stream);
    }
    return set_error(GDRN_ERR_ARG, "wgrad: unsupported n_tile=%d nsplit=%d", n_tile, nsplit);
}

static int pick_n_tile(int ntot, int nsplit) {
    if (nsplit == 1 && ntot % 256 == 0) return 256;
    if (ntot % 128 == 0) return 128;
    if (ntot % 64 == 0) return 64;
    return -1;
}

}  // namespace gdrn

using namespace gdrn;

// Workspace size query + K-split choice shared by conv and gemm wgrad.
static int choose_ksplit(int base_items, int kb_total, int requested) {
    if (requested > 0) return requested < kb_total ? requested : kb_total;
    // one full wave of CTAs (each CTA is one (tile, tap, K-split) work item and owns an SM: 1 CTA/SM by smem), with at
    // least 8 k-blocks per split so the pipeline fill / epilogue is amortised
    int ks = num_sms() / base_items;
    int max_ks = kb_total / 8;
    if (max_ks < 1) max_ks = 1;
    if (ks > max_ks) ks = max_ks;
    if (ks < 1) ks = 1;
    return ks;
}

extern "C" int gdrn_conv_wgrad(const void* dy_hi, const void* dy_lo, const void* x_hi, const void* x_lo, float* ws,
                               long ws_floats, long* ws_need_out, int* ksplit_out, int N, int H, int W, int Cin, int Cout, int KH, int KW,
                               int stride, int pad, int ksplit, int nsplit, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (nsplit != 1 && nsplit != 3) return set_error(GDRN_ERR_ARG, "conv_wgrad: nsplit must be 1 or 3");
    if (ws != nullptr && nsplit == 3 && (dy_lo == nullptr || x_lo == nullptr)) return set_error(GDRN_ERR_ARG, "conv_wgrad: lo planes missing");
    if (Cin % 64 || Cout % 64) return set_error(GDRN_ERR_ARG, "conv_wgrad: Cin/Cout must be multiples of 64");
    if (stride != 1 && stride != 2) return set_error(GDRN_ERR_ARG, "conv_wgrad: stride must be 1 or 2");
    const int Ho = H / stride, Wo = W / stride;
    if (Wo > 64 || 64 % Wo != 0) return set_error(GDRN_ERR_ARG, "conv_wgrad: unsupported output width %d", Wo);
    int THk = 64 / Wo;
    if (THk > Ho) THk = Ho;
    const int TNk = 64 / (Wo * THk);
    if (Ho % THk != 0 || (N % TNk) != 0) return set_error(GDRN_ERR_ARG, "conv_wgrad: shape not tileable by 64 pixels");
    const long P = (long)N * Ho * Wo;
    if (P % 64 != 0) return set_error(GDRN_ERR_ARG, "conv_wgrad: N*Ho*Wo must be a multiple of 64");
    // Cin == 64 (layer1): a 64-wide N tile leaves the tensor core smem/ingress-bound; pack the KW taps of a filter row
    // along N instead (N = 192): one dY tile load feeds three taps, 3x fewer MMAs / A loads per FLOP
    const int tap_pack = (nsplit == 1 && Cin == 64 && stride == 1 && KW == 3) ? 1 : 0;
    const int n_tile = tap_pack ? 192 : pick_n_tile(Cin, nsplit);
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.mode = 1;
    p.tap_pack = tap_pack;
    p.items = tap_pack ? KH : KH * KW;
    p.ws_ld = KH * KW * Cin;
    p.Mvalid = Cout;
    p.Ntot = Cin;
    p.num_m_tiles = (Cout + 127) / 128;
    p.num_n_tiles = tap_pack ? 1 : Cin / n_tile;
    p.taps = KH * KW;
    p.kb_total = (int)(P / 64);
    p.ksplit = choose_ksplit(p.num_m_tiles * p.num_n_tiles * p.items, p.kb_total, ksplit);
    p.KW = KW;
    p.pad = pad;
    p.stride = stride;
    p.THk = THk;
    p.TNk = TNk;
    p.blocks_per_img = (TNk == 1) ? Ho / THk : 0;
    p.ws = ws;
    if (ksplit_out) *ksplit_out = p.ksplit;
    const long need = (long)p.ksplit * p.num_m_tiles * 128 * p.taps * Cin;
    if (ws_need_out) *ws_need_out = need;
    if (ws == nullptr) return 0;  // size query only
    if (ws_floats < need) return set_error(GDRN_ERR_ARG, "conv_wgrad: workspace too small (%ld < %ld floats)", ws_floats, need);
    const int npl = nsplit == 1 ? 1 : 2;
    const void* dys[2] = {dy_hi, dy_lo};
    const void* xs[2] = {x_hi, x_lo};
    for (int pl = 0; pl < npl; ++pl) {
        uint64_t adims[2] = {(uint64_t)Cout, (uint64_t)P};
        uint64_t astr[1] = {(uint64_t)Cout * 2};
        uint32_t abox[2] = {64, 64};
        if (make_tmap(&p.tmA[pl], dys[pl], 2, adims, astr, abox)) return GDRN_ERR_CUDA;
        const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(xs[pl]);
        for (int ph = 0; ph < (stride == 2 ? 4 : 1); ++ph) {
            const int phh = ph >> 1, phw = ph & 1;
            uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)N};
            uint64_t strides[3] = {(uint64_t)stride * Cin * 2, (uint64_t)stride * W * Cin * 2, (uint64_t)H * W * Cin * 2};
            uint32_t box[4] = {64, (uint32_t)Wo, (uint32_t)THk, (uint32_t)TNk};
            if (make_tmap(&p.tmB[pl][ph], xb + ((size_t)phh * W + phw) * Cin, 4, dims, strides, box)) return GDRN_ERR_CUDA;
        }
    }
    return dispatch_wgrad(p, n_tile, nsplit, stream);
}

// dW[M][Ntot] = sum_p A[p][M] * B[p][Ntot]   (A = dY [P][M], B = X [P][Ntot]; P zero-padded to 64 by TMA)
extern "C" int gdrn_gemm_wgrad(const void* dy_hi, const void* dy_lo, const void* x_hi, const void* x_lo, float* ws,
                               long ws_floats, long* ws_need_out, int* ksplit_out, long P, int M, int Ntot, int ksplit, int nsplit,
                               void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (nsplit != 1 && nsplit != 3) return set_error(GDRN_ERR_ARG, "gemm_wgrad: nsplit must be 1 or 3");
    if (ws != nullptr && nsplit == 3 && (dy_lo == nullptr || x_lo == nullptr)) return set_error(GDRN_ERR_ARG, "gemm_wgrad: lo planes missing");
    if (M % 8 || Ntot % 64) return set_error(GDRN_ERR_ARG, "gemm_wgrad: M %% 8 and Ntot %% 64 required");
    const int n_tile = pick_n_tile(Ntot, nsplit);
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.mode = 0;
    p.Mvalid = M;
    p.Ntot = Ntot;
    p.num_m_tiles = (M + 127) / 128;
    p.num_n_tiles = Ntot / n_tile;
    p.taps = 1;
    p.items = 1;
    p.ws_ld = Ntot;
    p.kb_total = (int)((P + 63) / 64);
    p.ksplit = choose_ksplit(p.num_m_tiles * p.num_n_tiles, p.kb_total, ksplit);
    p.ws = ws;
    if (ksplit_out) *ksplit_out = p.ksplit;
    const long need = (long)p.ksplit * p.num_m_tiles * 128 * Ntot;
    if (ws_need_out) *ws_need_out = need;
    if (ws == nullptr) return 0;
    if (ws_floats < need) return set_error(GDRN_ERR_ARG, "gemm_wgrad: workspace too small (%ld < %ld floats)", ws_floats, need);
    const int npl = nsplit == 1 ? 1 : 2;
    const void* dys[2] = {dy_hi, dy_lo};
    const void* xs[2] = {x_hi, x_lo};
    for (int pl = 0; pl < npl; ++pl) {
        uint64_t adims[2] = {(uint64_t)M, (uint64_t)P};
        uint64_t astr[1] = {(uint64_t)M * 2};
        uint32_t abox[2] = {64, 64};
        if (make_tmap(&p.tmA[pl], dys[pl], 2, adims, astr, abox)) return GDRN_ERR_CUDA;
        uint64_t bdims[2] = {(uint64_t)Ntot, (uint64_t)P};
        uint64_t bstr[1] = {(uint64_t)Ntot * 2};
        if (make_tmap(&p.tmB[pl][0], xs[pl], 2, bdims, bstr, abox)) return GDRN_ERR_CUDA;
    }
    return dispatch_wgrad(p, n_tile, nsplit, stream);
}
