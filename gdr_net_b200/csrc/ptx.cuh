// sm_90a PTX wrappers used by the GEMM kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma fences and
// shared-memory matrix descriptors (the MMA itself is in wgmma.cuh).  Hand-written inline PTX; the descriptor
// layout follows the PTX ISA "matrix descriptor format" table of the wgmma section.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gdrn {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded spin: a broken pipeline traps (=> launch error surfaced to the host) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 22)) { __trap(); }
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}

// One lane of a converged warp (elect.sync): lets the producer / issuer loops run warp-uniformly (operands stay in uniform
// registers) while the asynchronous instruction itself is issued once.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// Lean variants for the single-thread producer / issuer loops: every operand is a precomputed 32-bit shared address or a
// 64-bit tensor-map / descriptor value, so nothing is converted or rebuilt on the per-k-block critical path.
__device__ __forceinline__ void mbar_wait_u32(uint32_t bar, uint32_t parity) {
    uint32_t spins = 0, ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (!ok && ++spins > (1u << 22)) __trap();
    } while (!ok);
}
__device__ __forceinline__ void mbar_arrive_expect_tx_u32(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d_u32(uint32_t dst, uint64_t tmap, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d_u32(uint32_t dst, uint64_t tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// TMA store of a box from shared memory (swizzled like the tensor map) to global memory; rows / columns outside the map's extent
// are not written.  Completion is tracked per issuing thread by bulk groups: `bulk_wait_group_read<N>` returns once the shared
// memory of all but the N most recent groups has been read (the staging buffer may be reused), `bulk_wait_group<N>` once their
// writes are done.  The generic-proxy writes that fill the box must be made visible with fence_proxy_async() first.
__device__ __forceinline__ void tma_store_2d_u32(uint64_t tmap, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap), "r"(src), "r"(c0),
                 "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Named barrier `id` (1..15; 0 is __syncthreads) over `threads` threads, a multiple of 32.
template <int ID, int THREADS>
__device__ __forceinline__ void named_bar_sync() {
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// ---------------------------------------------------------------- programmatic dependent launch
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor in the stream is
// still running; `pdl_wait` blocks until that predecessor has COMPLETED and its memory is visible.  Everything before it
// (barrier init, descriptor prefetch) overlaps the predecessor's tail.  `pdl_launch_dependents` lets the NEXT
// kernel of the stream begin that early start; it is always safe because the next kernel protects itself with its own wait.
// Both are no-ops when the launch carries no programmatic dependency.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// First statement of every elementwise / pack kernel that launch_pdl() (gdrn_internal.h) may start early.
__device__ __forceinline__ void pdl_ew_entry() {
#if !defined(GDRN_PDL_EW_NO_TRIGGER)
    pdl_launch_dependents();
#endif
    pdl_wait();
}

// ---------------------------------------------------------------- wgmma
// An MMA issued by a warpgroup reads its shared-memory operands asynchronously: fence before the first MMA that uses
// register accumulators written by ordinary instructions, commit the issued MMAs as one group, and wait until at most
// N groups are pending before their accumulators are read or their operand stage is handed back to the producer.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across an asynchronous MMA.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor of wgmma (PTX ISA "matrix descriptor format"):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4 | [62,64) swizzle: 1 = 128B
// K-major SW128 tile  [rows][64 16-bit = 128 B]: 8-row groups are 1024 B apart (SBO); LBO unused (=1).  A 16-wide k-step
//   advances the start address by 32 B (+2 in the descriptor).
// MN-major SW128 tile [k rows][64 16-bit = 128 B] per 64-wide MN chunk: SBO = 1024 B between 8-k-row groups, LBO = byte
//   distance between consecutive 64-element MN chunks.  A 16-deep k-step advances by 16 rows = 2048 B (+128).
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ---------------------------------------------------------------- 16-bit storage format of the (hi, lo) planes
// GDRN_STORE_F16 = 0: hi = bf16(x),  lo = bf16(x - hi)               (8 + 8 bits; fp32 exponent range)
// GDRN_STORE_F16 = 1: hi = fp16(x),  lo = fp16((x - hi) * 2^11)       (11 + 11 bits: the single-plane mode has the
//     mantissa of TF32 -- what cuDNN uses for the reference's fp32 convolutions -- and the two-plane mode 22 bits.
//     The scaled residual has the magnitude of x itself, so it needs no extra exponent range; the scale is divided
//     out exactly in the GEMM epilogues (cross-term accumulator) and in load8().  Gradients are kept in range by a
//     static loss scale applied by the engine (Engine.grad_scale), like AMP's GradScaler in the reference's configs.)
// Both planes must share one format: one wgmma multiplies operands of a single 16-bit type (wgmma.cuh).
#ifndef GDRN_STORE_F16
#define GDRN_STORE_F16 0
#endif
#if GDRN_STORE_F16
constexpr float kLoScale = 2048.f;
constexpr float kLoInvScale = 1.f / 2048.f;
__device__ __forceinline__ uint32_t pack_hi2(float a, float b) {  // a -> low half, b -> high half
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
__device__ __forceinline__ void unpack_hi2(uint32_t w, float& a, float& b) {
    asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}" : "=f"(a), "=f"(b) : "r"(w));
}
#else
constexpr float kLoScale = 1.f;
constexpr float kLoInvScale = 1.f;
__device__ __forceinline__ uint32_t pack_hi2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
__device__ __forceinline__ void unpack_hi2(uint32_t w, float& a, float& b) {
    a = __uint_as_float(w << 16);
    b = __uint_as_float(w & 0xffff0000u);
}
#endif
__device__ __forceinline__ uint32_t pack_lo2(float ra, float rb) { return pack_hi2(ra * kLoScale, rb * kLoScale); }
__device__ __forceinline__ void unpack_lo2(uint32_t w, float& a, float& b) {
    unpack_hi2(w, a, b);
    a *= kLoInvScale;
    b *= kLoInvScale;
}
// (a, b) -> packed hi pair and packed lo pair (residuals after rounding to the hi format)
__device__ __forceinline__ void split2(float a, float b, uint32_t& h, uint32_t& l) {
    h = pack_hi2(a, b);
    float ha, hb;
    unpack_hi2(h, ha, hb);
    l = pack_lo2(a - ha, b - hb);
}
// scalar versions (weight packing): 16-bit patterns
__device__ __forceinline__ void split1(float x, uint16_t& h, uint16_t& l) {
    uint32_t hh, ll;
    split2(x, 0.f, hh, ll);
    h = (uint16_t)(hh & 0xffffu);
    l = (uint16_t)(ll & 0xffffu);
}

}  // namespace gdrn
