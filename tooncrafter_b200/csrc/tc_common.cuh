// tooncrafter_b200 — shared device-side primitives for the sm_90a kernels.
//
// Thin inline-PTX wrappers around the Hopper async machinery: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (warpgroup MMA with shared-memory descriptors), clusters and programmatic dependent launch.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

namespace tc {

// ---------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .b32 rx;\n\t"
        ".reg .pred px;\n\t"
        "elect.sync rx|px, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, px;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void lds128(uint32_t addr, float4& v) {
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (-> cudaErrorLaunchFailure) instead of hanging the GPU.  No printf here: the MMA
// warpgroups wait inside their wgmma k-loop, and any function call there (printf, assert) makes ptxas serialise every
// wgmma.mma_async of the kernel (warning C7510).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s at 2 GHz
    }
}

// ---------------------------------------------------------------------------------------------
// TMA tile loads (global -> shared), completion on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma: warpgroup MMA (sm_90a), A and B from shared memory, fp32 accumulators in registers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kN>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kN) : "memory");
}
// D[64 x N] += A[64 x 16] * B[16 x N], N = 32 kNJ: fp16 operands, both K-major in shared memory; this thread's 16 kNJ
// accumulators (row = 16 * warp + lane / 4 + 8 * ((i >> 1) & 1), column = 8 * (i >> 2) + 2 * (lane % 4) + (i & 1)).
// One instruction per k16 step reads A once for all N columns.  The operand lists are spelled out by the macros below
// (asm templates are string literals); operands 0 .. 16 kNJ - 1 are the accumulators, then the two descriptors.
template <int kNJ>
__device__ __forceinline__ void wgmma_m64nNk16(float (&d)[16 * kNJ], uint64_t desc_a, uint64_t desc_b);

#define TC_WG_R16_0 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define TC_WG_R16_1 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define TC_WG_R16_2 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define TC_WG_R16_3 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define TC_WG_R16_4 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define TC_WG_R16_5 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define TC_WG_R16_6 "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
#define TC_WG_R16_7 "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define TC_WG_REGS_1 TC_WG_R16_0
#define TC_WG_REGS_2 TC_WG_REGS_1 ", " TC_WG_R16_1
#define TC_WG_REGS_3 TC_WG_REGS_2 ", " TC_WG_R16_2
#define TC_WG_REGS_4 TC_WG_REGS_3 ", " TC_WG_R16_3
#define TC_WG_REGS_5 TC_WG_REGS_4 ", " TC_WG_R16_4
#define TC_WG_REGS_6 TC_WG_REGS_5 ", " TC_WG_R16_5
#define TC_WG_REGS_7 TC_WG_REGS_6 ", " TC_WG_R16_6
#define TC_WG_REGS_8 TC_WG_REGS_7 ", " TC_WG_R16_7
#define TC_WG_ACC16(o)                                                                                                  \
    "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]),     \
        "+f"(d[o + 7]), "+f"(d[o + 8]), "+f"(d[o + 9]), "+f"(d[o + 10]), "+f"(d[o + 11]), "+f"(d[o + 12]),              \
        "+f"(d[o + 13]), "+f"(d[o + 14]), "+f"(d[o + 15])
#define TC_WG_ACC_1 TC_WG_ACC16(0)
#define TC_WG_ACC_2 TC_WG_ACC_1, TC_WG_ACC16(16)
#define TC_WG_ACC_3 TC_WG_ACC_2, TC_WG_ACC16(32)
#define TC_WG_ACC_4 TC_WG_ACC_3, TC_WG_ACC16(48)
#define TC_WG_ACC_5 TC_WG_ACC_4, TC_WG_ACC16(64)
#define TC_WG_ACC_6 TC_WG_ACC_5, TC_WG_ACC16(80)
#define TC_WG_ACC_7 TC_WG_ACC_6, TC_WG_ACC16(96)
#define TC_WG_ACC_8 TC_WG_ACC_7, TC_WG_ACC16(112)
// NJ, N = 32 NJ, and the operand numbers of the two descriptors (16 NJ, 16 NJ + 1)
#define TC_WGMMA_M64NK16(NJ, N, DA, DB)                                                                                 \
    template <>                                                                                                         \
    __device__ __forceinline__ void wgmma_m64nNk16<NJ>(float(&d)[16 * NJ], uint64_t desc_a, uint64_t desc_b) {          \
        asm volatile("{\n\t"                                                                                            \
                     ".reg .pred p;\n\t"                                                                                \
                     "setp.ne.b32 p, 1, 0;\n\t"                                                                         \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 "                                          \
                     "{" TC_WG_REGS_##NJ "}, %" #DA ", %" #DB ", p, 1, 1, 0, 0;\n\t"                                    \
                     "}\n"                                                                                              \
                     : TC_WG_ACC_##NJ                                                                                   \
                     : "l"(desc_a), "l"(desc_b));                                                                       \
    }
TC_WGMMA_M64NK16(1, 32, 16, 17)
TC_WGMMA_M64NK16(2, 64, 32, 33)
TC_WGMMA_M64NK16(3, 96, 48, 49)
TC_WGMMA_M64NK16(4, 128, 64, 65)
TC_WGMMA_M64NK16(5, 160, 80, 81)
TC_WGMMA_M64NK16(6, 192, 96, 97)
TC_WGMMA_M64NK16(7, 224, 112, 113)
TC_WGMMA_M64NK16(8, 256, 128, 129)
#undef TC_WGMMA_M64NK16

// ---- programmatic dependent launch: every kernel of this library is launched with the programmatic-stream-serialization
// attribute (tc_host::launch), lets its successor's CTAs start early (launch_dependents) and must execute pdl_wait()
// before its first access to global memory a predecessor may have written — and EVERY kernel must execute it, otherwise
// completion of kernel N would no longer imply completion of kernel N-1 for kernel N+1.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- TMA stores (shared -> global, bulk async group completion) ---------------------------------------
__device__ __forceinline__ void tma_store_4d(const void* smem_src, const void* tmap, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
        :
        : "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the newest kN groups have finished READING their shared-memory source (buffer reusable)
template <int kN>
__device__ __forceinline__ void bulk_wait_group_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kN) : "memory");
}
template <int kN>
__device__ __forceinline__ void bulk_wait_group() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(kN) : "memory");
}
// ---------------------------------------------------------------------------------------------
// clusters
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same smem offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    asm volatile(
        "{\n\t"
        ".reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(cta)
        : "memory");
}
// ---------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, 128-byte swizzle, K-major rows of 128 bytes packed densely (8-row swizzle
// atoms of 1024 B, as TMA writes a box whose inner extent is 64 halfs with CU_TENSOR_MAP_SWIZZLE_128B).
//   bits [0,14) start address >> 4     bits [16,30) leading byte offset >> 4 (unused for swizzled K-major)
//   bits [32,46) stride byte offset >> 4 (1024 B between 8-row groups)     bits [62,64) layout (1 = SWIZZLE_128B)
// Advancing K by 16 halfs inside the swizzle row adds 32 bytes (+2) to the start address field.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

// erf by Abramowitz & Stegun 7.1.28: 1 - (1 + a1 x + ... + a6 x^6)^-16, |err| <= 3e-7: 6 FMA + 4 squarings + ONE
// MUFU (rcp.approx) instead of libm erff's ~25-instruction path; the GEGLU epilogue at K = 320 is ALU-bound.
// (A rcp + ex2 variant, 7.1.26, was MUFU-bound and 1.5x slower than libm.)
__device__ __forceinline__ float erf_fast(float x) {
    const float ax = fabsf(x);
    float t = fmaf(ax, 0.0000430638f, 0.0002765672f);
    t = fmaf(t, ax, 0.0001520143f);
    t = fmaf(t, ax, 0.0092705272f);
    t = fmaf(t, ax, 0.0422820123f);
    t = fmaf(t, ax, 0.0705230784f);
    t = fmaf(t, ax, 1.0f);
    t *= t;
    t *= t;
    t *= t;
    t *= t;
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(t));
    return copysignf(1.0f - r, x);
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erf_fast(x * 0.70710678118654752f)); }

// a * GELU(x): the cheap form of the GEGLU product.
// GELU(x) = x * Phi(x) with Phi(x) = 1 - h for x >= 0 and h for x < 0, h = 0.5 * (1 + a1 z + ... + a6 z^6)^-16,
// z = |x| / sqrt(2): the same A&S 7.1.28 polynomial with 2^(-i/2) (the x/sqrt(2)) and 2^(1/16) (the 0.5) folded into its
// coefficients: 6 FFMA + 4 FMUL + 1 MUFU + FADD + FSEL + 2 FMUL, |GELU error| <= 8e-7.
__device__ __forceinline__ float geglu_mul(float a, float x) {
    const float ax = fabsf(x);
    float t = fmaf(ax, 5.6212996640e-06f, 5.1055209009e-05f);
    t = fmaf(t, ax, 3.9686137011e-05f);
    t = fmaf(t, ax, 3.4227392389e-03f);
    t = fmaf(t, ax, 2.2076998457e-02f);
    t = fmaf(t, ax, 5.2075163037e-02f);
    t = fmaf(t, ax, 1.0442737824e+00f);
    t *= t;
    t *= t;
    t *= t;
    t *= t;
    float h;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(h) : "f"(t));
    const float phi = x >= 0.f ? 1.0f - h : h;
    return (a * x) * phi;
}


}  // namespace tc
