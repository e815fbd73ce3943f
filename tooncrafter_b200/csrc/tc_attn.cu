// tooncrafter_b200 — attention kernels.
//
//  tc_attention           fused softmax(QK^T)V, head dim 64, one or two key/value segments (each with its own softmax,
//                         outputs summed), mma.sync m16n8k16 with fp32 accumulators and an fp32 online softmax; one
//                         segment may also take head dim 80 (OpenCLIP ViT-H/14 vision tower) and a causal mask (its
//                         text tower).
//  tc_attention_wide      the same kernel for one head of up to 512 channels (VAE mid-block attention): scores stay
//                         on chip; each CTA produces 256, 128 or 64 of the value channels (the widest that divides D).
//  tc_temporal_attention  temporal self-attention over T <= 64 frames, one (pixel, head) per warp, mma.sync 16x8x16
//                         (HBM-bound): one kernel for T <= 16, one for 16 < T <= 64.
//  tc_softmax_rows        row softmax over a stored score matrix.
//
// Reference sites: lvdm/modules/attention.py:81-209,365-412; lvdm/models/autoencoder_dualref.py:172-200,270-341.
#include <stdlib.h>
#include "tc_common.cuh"
#include "tc_host.h"

namespace {

__device__ __forceinline__ uint32_t pack_h2(float x, float y) {
    __half2 h = __floats2half2_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&h);
}
// (x, y) = hi + lo with hi = fp16(x, y) and lo = fp16 of the rounding residual
__device__ __forceinline__ void split_h2(float x, float y, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 f = __half22float2(h);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = pack_h2(x - f.x, y - f.y);
}
__device__ __forceinline__ void mma_m16n8k16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// 16-byte global -> shared copy, zero-filled when !ok
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int kN>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(kN) : "memory"); }

// ===================================================================================== fused attention
// Flash-style: a CTA of 4 warps takes 64 query rows (16 per warp) of one (batch, head, value chunk); key tiles of 64
// rows are staged in shared memory (K and V loads in separate cp.async groups, so S = Q K^T runs while V arrives).
// Rows of D halfs are stored with their 16-byte chunks XOR-swizzled by (row & 7) so ldmatrix rows hit distinct banks.
// The XOR needs 8k chunks per row; 80-wide rows (10 chunks) use a padded row stride of 11 chunks instead (tile_off).
constexpr int kFaRows = 64;
constexpr int kFaKeys = 64;
constexpr int kFaThreads = 128;

struct FaSeg {
    const __half* k;
    const __half* v;
    long long ldk, ldv;
    int Lk, kv_div;        // K/V batch = query batch / kv_div
};
struct FaParams {
    const __half* q;
    long long ldq;
    int Lq, heads;
    int D;                 // q / k width per head
    int DV, nv;            // value columns per CTA, value chunks per head (D = DV * nv)
    int n_seg;
    FaSeg seg[2];
    __half* out;
    long long ldo;
    float scale_log2;
    int split_p;
};

// byte offset of 16-byte chunk c of row r in a swizzled tile with `cpr` chunks per row
__device__ __forceinline__ uint32_t swz(int r, int c, int cpr) { return (uint32_t)((r * cpr + (c ^ (r & 7))) << 4); }

// Tile layout of the head-dim-80 instance (10 chunks per row): rows padded to 11 chunks (176 bytes), no XOR.  An
// ldmatrix phase reads one 16-byte chunk from each of 8 consecutive rows r..r+7 at the same column; their chunk indices
// 11 r + c fall in bank groups (11 r + c) mod 8, and since 11 is odd, r -> 11 r mod 8 is a bijection on 8 consecutive
// rows: the 8 reads hit 8 distinct 16-byte bank groups (conflict-free).
constexpr int kPadCpr = 11;
template <int kDV>
__device__ __forceinline__ uint32_t tile_off(int r, int c, int cpr) {
    if constexpr (kDV == 80) return (uint32_t)((r * kPadCpr + c) << 4);
    else return swz(r, c, cpr);
}
// shared-memory bytes of one tile of `rows` rows of D halfs
__host__ __device__ constexpr int tile_bytes(int rows, int D) { return D == 80 ? rows * kPadCpr * 16 : rows * D * 2; }

// kTwoSeg: up to two key/value segments, each with its own softmax, outputs summed (a second accumulator set).
// kDV = 80: head dim 80 for q / k and v (single segment).  kCausal: key j is masked for query i when j > i, and key
// tiles wholly above the diagonal of this CTA's query rows are skipped.
template <int kDV, bool kTwoSeg, bool kCausal>
__global__ void __launch_bounds__(kFaThreads) flash_attn_kernel(const FaParams p) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    extern __shared__ __align__(128) uint8_t fa_smem[];
    const int D = p.D, cq = D / 8;                 // 16-byte chunks per q / k row
    constexpr int cv = kDV / 8;                    // 16-byte chunks per v row
    const uint32_t sQ = tc::smem_u32(fa_smem);
    const uint32_t sK = sQ + (uint32_t)(kDV == 80 ? tile_bytes(kFaRows, 80) : kFaRows * D * 2);
    const uint32_t sV = sK + (uint32_t)(kDV == 80 ? tile_bytes(kFaKeys, 80) : kFaKeys * D * 2);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q0 = blockIdx.x * kFaRows;
    const int head = blockIdx.y / p.nv, vchunk = blockIdx.y - head * p.nv;
    const int b = blockIdx.z;
    const int qk_col = head * D, v_col = head * D + vchunk * kDV;

    // ---- Q tile
    for (int i = tid; i < kFaRows * cq; i += kFaThreads) {
        const int r = i / cq, c = i - r * cq;
        const bool ok = q0 + r < p.Lq;
        const __half* src = p.q + ((long long)b * p.Lq + (ok ? q0 + r : 0)) * p.ldq + qk_col + c * 8;
        cp_async16(sQ + tile_off<kDV>(r, c, cq), src, ok);
    }
    cp_async_commit();

    float ot[kTwoSeg ? kDV / 8 : 1][4];   // sum over the segments (two-segment form only)
#pragma unroll
    for (int j = 0; j < (kTwoSeg ? kDV / 8 : 1); ++j) ot[j][0] = ot[j][1] = ot[j][2] = ot[j][3] = 0.f;
    float o[kDV / 8][4];
    const int g = lane >> 2, t4 = lane & 3;

    for (int s = 0; s < (kTwoSeg ? p.n_seg : 1); ++s) {
        const FaSeg sg = p.seg[s];
        const long long kvb = b / sg.kv_div;
#pragma unroll
        for (int j = 0; j < kDV / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
        // causal: keys beyond this CTA's last query row are masked for every row of the CTA
        const int k_end = kCausal ? min(sg.Lk, q0 + kFaRows) : sg.Lk;
        for (int k0 = 0; k0 < k_end; k0 += kFaKeys) {
            __syncthreads();   // every warp is done with the previous K / V tile
            for (int i = tid; i < kFaKeys * cq; i += kFaThreads) {
                const int r = i / cq, c = i - r * cq;
                const bool ok = k0 + r < sg.Lk;
                cp_async16(sK + tile_off<kDV>(r, c, cq), sg.k + (kvb * sg.Lk + (ok ? k0 + r : 0)) * sg.ldk + qk_col + c * 8, ok);
            }
            cp_async_commit();
            for (int i = tid; i < kFaKeys * cv; i += kFaThreads) {
                const int r = i / cv, c = i - r * cv;
                const bool ok = k0 + r < sg.Lk;
                cp_async16(sV + tile_off<kDV>(r, c, cv), sg.v + (kvb * sg.Lk + (ok ? k0 + r : 0)) * sg.ldv + v_col + c * 8, ok);
            }
            cp_async_commit();
            cp_async_wait<1>();   // Q and K have landed
            __syncthreads();

            // ---- S = Q K^T for this warp's 16 rows x 64 keys
            float sc[8][4];
#pragma unroll
            for (int j = 0; j < 8; ++j) sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
            for (int kk = 0; kk < D / 16; ++kk) {
                uint32_t a[4];
                ldsm_x4(sQ + tile_off<kDV>(warp * 16 + (lane & 15), 2 * kk + (lane >> 4), cq), a[0], a[1], a[2], a[3]);
#pragma unroll
                for (int np = 0; np < 4; ++np) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4(sK + tile_off<kDV>(np * 16 + (lane & 7) + ((lane >> 4) << 3), 2 * kk + ((lane >> 3) & 1), cq), b0, b1, b2, b3);
                    mma_m16n8k16(sc[2 * np], a, b0, b1);
                    mma_m16n8k16(sc[2 * np + 1], a, b2, b3);
                }
            }
            // ---- online softmax (rows g and g + 8 of the warp; a row lives in the 4 lanes of a quad)
            float mx0 = m0, mx1 = m1;
            const int qr0 = q0 + warp * 16 + g;    // query rows of sc[.][0..1] and sc[.][2..3]: qr0, qr0 + 8
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int key = k0 + 8 * j + 2 * t4 + i;
                    const bool key_ok = key < sg.Lk;
                    const bool ok0 = key_ok && (!kCausal || key <= qr0);
                    const bool ok1 = key_ok && (!kCausal || key <= qr0 + 8);
                    sc[j][i] = ok0 ? sc[j][i] * p.scale_log2 : -INFINITY;
                    sc[j][2 + i] = ok1 ? sc[j][2 + i] * p.scale_log2 : -INFINITY;
                    mx0 = fmaxf(mx0, sc[j][i]);
                    mx1 = fmaxf(mx1, sc[j][2 + i]);
                }
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            const float al0 = exp2f(m0 - mx0), al1 = exp2f(m1 - mx1);   // 0 on the first tile (m = -inf)
            m0 = mx0;
            m1 = mx1;
            l0 *= al0;
            l1 *= al1;
#pragma unroll
            for (int j = 0; j < kDV / 8; ++j) {
                o[j][0] *= al0;
                o[j][1] *= al0;
                o[j][2] *= al1;
                o[j][3] *= al1;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                sc[j][0] = exp2f(sc[j][0] - m0);
                sc[j][1] = exp2f(sc[j][1] - m0);
                sc[j][2] = exp2f(sc[j][2] - m1);
                sc[j][3] = exp2f(sc[j][3] - m1);
                l0 += sc[j][0] + sc[j][1];
                l1 += sc[j][2] + sc[j][3];
            }
            cp_async_wait<0>();   // V has landed
            __syncthreads();
            // ---- O += P V (P as the A operand straight from the score fragments)
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) {
                uint32_t pa[4], pl[4];
                split_h2(sc[2 * kb][0], sc[2 * kb][1], pa[0], pl[0]);
                split_h2(sc[2 * kb][2], sc[2 * kb][3], pa[1], pl[1]);
                split_h2(sc[2 * kb + 1][0], sc[2 * kb + 1][1], pa[2], pl[2]);
                split_h2(sc[2 * kb + 1][2], sc[2 * kb + 1][3], pa[3], pl[3]);
                const int mrow = kb * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
                for (int nd = 0; nd < kDV / 8; nd += 2) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4_t(sV + tile_off<kDV>(mrow, nd + (lane >> 4), cv), b0, b1, b2, b3);
                    if (p.split_p) {
                        mma_m16n8k16(o[nd], pl, b0, b1);
                        mma_m16n8k16(o[nd + 1], pl, b2, b3);
                    }
                    mma_m16n8k16(o[nd], pa, b0, b1);
                    mma_m16n8k16(o[nd + 1], pa, b2, b3);
                }
            }
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
#pragma unroll
        for (int j = 0; j < kDV / 8; ++j) {
            o[j][0] *= inv0;
            o[j][1] *= inv0;
            o[j][2] *= inv1;
            o[j][3] *= inv1;
            if constexpr (kTwoSeg) {
                ot[j][0] += o[j][0];
                ot[j][1] += o[j][1];
                ot[j][2] += o[j][2];
                ot[j][3] += o[j][3];
            }
        }
    }
    if constexpr (kTwoSeg) {
#pragma unroll
        for (int j = 0; j < kDV / 8; ++j) {
            o[j][0] = ot[j][0];
            o[j][1] = ot[j][1];
            o[j][2] = ot[j][2];
            o[j][3] = ot[j][3];
        }
    }
    const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
    __half* o0p = p.out + ((long long)b * p.Lq + r0) * p.ldo + v_col + 2 * t4;
    __half* o1p = p.out + ((long long)b * p.Lq + r1) * p.ldo + v_col + 2 * t4;
#pragma unroll
    for (int j = 0; j < kDV / 8; ++j) {
        if (r0 < p.Lq) *reinterpret_cast<uint32_t*>(o0p + 8 * j) = pack_h2(o[j][0], o[j][1]);
        if (r1 < p.Lq) *reinterpret_cast<uint32_t*>(o1p + 8 * j) = pack_h2(o[j][2], o[j][3]);
    }
}

// ===================================================================================== temporal attention, T <= 16
// One warp per (batch, pixel, head): the whole problem is a 16 x 16 x 64 attention, far below a 64-row wgmma tile,
// and the kernel is HBM-bound (reads q, k, v once, writes o once).  S = Q K^T and O = P V use warp-level
// mma.sync.m16n8k16 with fragments loaded straight from global memory (Q, K) or via ldmatrix.trans from a
// swizzled 2 KiB smem tile (V); softmax in fp32 on the accumulator fragments.
__global__ void __launch_bounds__(128) temporal_attn_mma_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                                const __half* __restrict__ v, long long ld,
                                                                __half* __restrict__ out, long long ldo, int B, int T,
                                                                int P, int heads, float scale_log2) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    __shared__ __align__(128) uint8_t sV[4][16 * 128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t4 = lane & 3;
    const long long total = (long long)B * P * heads;
    const long long frame_stride = (long long)P * ld;       // elements between consecutive frames of one pixel
    uint8_t* sv = sV[warp];
    for (long long item = (long long)blockIdx.x * 4 + warp; item < total; item += (long long)gridDim.x * 4) {
        const int h = (int)(item % heads);
        const long long r = item / heads;
        const long long pix = r % P, b = r / P;
        const long long base = ((b * T) * P + pix) * ld + h * 64;   // frame 0 of this (b, pix, head)
        // ---- V tile -> smem (16-byte chunks, XOR-swizzled so ldmatrix rows hit distinct banks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int chunk = lane + 32 * i;
            const int row = chunk >> 3, c16 = chunk & 7;
            uint4 u = make_uint4(0u, 0u, 0u, 0u);
            if (row < T) u = *reinterpret_cast<const uint4*>(v + base + row * frame_stride + c16 * 8);
            *reinterpret_cast<uint4*>(sv + row * 128 + ((c16 ^ (row & 7)) << 4)) = u;
        }
        // ---- Q (A fragments) and K (B fragments) straight from global
        uint32_t qa[4][4], kb[2][4][2];
        const bool r0 = g < T, r1 = g + 8 < T;
        const __half* q0p = q + base + (long long)g * frame_stride;
        const __half* q1p = q + base + (long long)(g + 8) * frame_stride;
        const __half* k0p = k + base + (long long)g * frame_stride;
        const __half* k1p = k + base + (long long)(g + 8) * frame_stride;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const int c = 16 * ks + 2 * t4;
            qa[ks][0] = r0 ? *reinterpret_cast<const uint32_t*>(q0p + c) : 0u;
            qa[ks][1] = r1 ? *reinterpret_cast<const uint32_t*>(q1p + c) : 0u;
            qa[ks][2] = r0 ? *reinterpret_cast<const uint32_t*>(q0p + c + 8) : 0u;
            qa[ks][3] = r1 ? *reinterpret_cast<const uint32_t*>(q1p + c + 8) : 0u;
            kb[0][ks][0] = r0 ? *reinterpret_cast<const uint32_t*>(k0p + c) : 0u;
            kb[0][ks][1] = r0 ? *reinterpret_cast<const uint32_t*>(k0p + c + 8) : 0u;
            kb[1][ks][0] = r1 ? *reinterpret_cast<const uint32_t*>(k1p + c) : 0u;
            kb[1][ks][1] = r1 ? *reinterpret_cast<const uint32_t*>(k1p + c + 8) : 0u;
        }
        float sacc[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int i = 0; i < 4; ++i) sacc[nt][i] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) mma_m16n8k16(sacc[nt], qa[ks], kb[nt][ks][0], kb[nt][ks][1]);
        }
        // ---- softmax over the 16 keys of rows g and g + 8 (a row lives in the 4 lanes of a quad)
        float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const bool key_ok = (8 * nt + 2 * t4 + i) < T;
                sacc[nt][i] = key_ok ? sacc[nt][i] * scale_log2 : -INFINITY;
                sacc[nt][2 + i] = key_ok ? sacc[nt][2 + i] * scale_log2 : -INFINITY;
                m0 = fmaxf(m0, sacc[nt][i]);
                m1 = fmaxf(m1, sacc[nt][2 + i]);
            }
        }
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
        m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
        m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
        float l0 = 0.f, l1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                sacc[nt][i] = exp2f(sacc[nt][i] - m0);
                sacc[nt][2 + i] = exp2f(sacc[nt][2 + i] - m1);
                l0 += sacc[nt][i];
                l1 += sacc[nt][2 + i];
            }
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
        // P = hi + lo with both parts fp16: with only T <= 16 keys per query the fp16 rounding of P is not averaged
        // away, and the kernel is HBM-bound, so the second (residual) MMA is free
        uint32_t pa[4], pl[4];
        split_h2(sacc[0][0] * inv0, sacc[0][1] * inv0, pa[0], pl[0]);
        split_h2(sacc[0][2] * inv1, sacc[0][3] * inv1, pa[1], pl[1]);
        split_h2(sacc[1][0] * inv0, sacc[1][1] * inv0, pa[2], pl[2]);
        split_h2(sacc[1][2] * inv1, sacc[1][3] * inv1, pa[3], pl[3]);
        __syncwarp();
        // ---- O = P V, V fragments by ldmatrix.trans (two 8-wide d tiles per instruction)
        __half* o0p = out + ((b * T + g) * P + pix) * ldo + h * 64;
        __half* o1p = out + ((b * T + g + 8) * P + pix) * ldo + h * 64;
#pragma unroll
        for (int nd = 0; nd < 8; nd += 2) {
            // lane i supplies the row address of matrix i/8: matrices (k 0-7, nd), (k 8-15, nd), (k 0-7, nd+1), (k 8-15, nd+1)
            const int mrow = (lane & 7) + ((lane >> 3) & 1) * 8;
            const int mcol = nd + (lane >> 4);
            const uint32_t addr = tc::smem_u32(sv + mrow * 128 + ((mcol ^ (mrow & 7)) << 4));
            uint32_t b0, b1, b2, b3;
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                         : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3)
                         : "r"(addr));
            float oa[4] = {0.f, 0.f, 0.f, 0.f}, ob[4] = {0.f, 0.f, 0.f, 0.f};
            mma_m16n8k16(oa, pl, b0, b1);
            mma_m16n8k16(ob, pl, b2, b3);
            mma_m16n8k16(oa, pa, b0, b1);
            mma_m16n8k16(ob, pa, b2, b3);
            if (r0) {
                *reinterpret_cast<uint32_t*>(o0p + 8 * nd + 2 * t4) = pack_h2(oa[0], oa[1]);
                *reinterpret_cast<uint32_t*>(o0p + 8 * (nd + 1) + 2 * t4) = pack_h2(ob[0], ob[1]);
            }
            if (r1) {
                *reinterpret_cast<uint32_t*>(o1p + 8 * nd + 2 * t4) = pack_h2(oa[2], oa[3]);
                *reinterpret_cast<uint32_t*>(o1p + 8 * (nd + 1) + 2 * t4) = pack_h2(ob[2], ob[3]);
            }
        }
        __syncwarp();   // smem V tile is reused by the next item
    }
}

// ===================================================================================== temporal attention, 16 < T <= 64
// One warp per (batch, pixel, head), kTiles = ceil(T / 16) tiles of 16 frames.  K and V (T x 64 fp16 each, up to
// 8 KiB) are staged by cp.async into this warp's swizzled smem tiles, zero-filled past frame T; K feeds the B operand
// of S = Q K^T by ldmatrix, V the B operand of O = P V by ldmatrix.trans.  Each 16-row query tile computes its scores
// against all T keys at once, so the softmax is exact (no running maximum), in fp32 on the accumulator fragments.
// Dynamic smem: 4 warps x (K + V) x kTiles * 2 KiB, room for 6, 4 or 3 CTAs per SM at kTiles = 2, 3, 4; the register
// bound asks for 5 (6 would spill), 4 and 3.
template <int kTiles>
__global__ void __launch_bounds__(128, kTiles == 2 ? 5 : 12 / kTiles) temporal_attn_mma64_kernel(const __half* __restrict__ q,
                                                                  const __half* __restrict__ k,
                                                                  const __half* __restrict__ v, long long ld,
                                                                  __half* __restrict__ out, long long ldo, int B, int T,
                                                                  int P, int heads, float scale_log2) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    constexpr int kRows = 16 * kTiles;
    constexpr int kTileBytes = kRows * 128;
    extern __shared__ __align__(128) uint8_t tsmem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t4 = lane & 3;
    const uint32_t sK = tc::smem_u32(tsmem) + (uint32_t)(warp * 2 * kTileBytes);
    const uint32_t sV = sK + (uint32_t)kTileBytes;
    const long long total = (long long)B * P * heads;
    const long long frame_stride = (long long)P * ld;       // elements between consecutive frames of one pixel
    for (long long item = (long long)blockIdx.x * 4 + warp; item < total; item += (long long)gridDim.x * 4) {
        const int h = (int)(item % heads);
        const long long r = item / heads;
        const long long pix = r % P, b = r / P;
        const long long base = ((b * T) * P + pix) * ld + h * 64;   // frame 0 of this (b, pix, head)
        // ---- K, then V -> smem (two cp.async groups: S runs while V lands); frames >= T are zeros
#pragma unroll
        for (int i = 0; i < kRows * 8 / 32; ++i) {
            const int chunk = lane + 32 * i, row = chunk >> 3, c16 = chunk & 7;
            const bool ok = row < T;
            cp_async16(sK + swz(row, c16, 8), k + base + (ok ? row * frame_stride : 0) + c16 * 8, ok);
        }
        cp_async_commit();
#pragma unroll
        for (int i = 0; i < kRows * 8 / 32; ++i) {
            const int chunk = lane + 32 * i, row = chunk >> 3, c16 = chunk & 7;
            const bool ok = row < T;
            cp_async16(sV + swz(row, c16, 8), v + base + (ok ? row * frame_stride : 0) + c16 * 8, ok);
        }
        cp_async_commit();
        for (int mt = 0; mt < kTiles; ++mt) {
            // ---- Q (A fragments) of query frames 16 mt + g and 16 mt + g + 8, straight from global
            const int q0 = 16 * mt + g, q1 = q0 + 8;
            const bool r0 = q0 < T, r1 = q1 < T;
            const __half* q0p = q + base + (long long)q0 * frame_stride;
            const __half* q1p = q + base + (long long)q1 * frame_stride;
            uint32_t qa[4][4];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const int c = 16 * ks + 2 * t4;
                qa[ks][0] = r0 ? *reinterpret_cast<const uint32_t*>(q0p + c) : 0u;
                qa[ks][1] = r1 ? *reinterpret_cast<const uint32_t*>(q1p + c) : 0u;
                qa[ks][2] = r0 ? *reinterpret_cast<const uint32_t*>(q0p + c + 8) : 0u;
                qa[ks][3] = r1 ? *reinterpret_cast<const uint32_t*>(q1p + c + 8) : 0u;
            }
            if (mt == 0) {
                cp_async_wait<1>();   // K has landed
                __syncwarp();
            }
            // ---- S = Q K^T over all 16 kTiles keys (n tiles 2 np, 2 np + 1 from one ldmatrix.x4 per 16 d)
            float sacc[2 * kTiles][4];
#pragma unroll
            for (int nt = 0; nt < 2 * kTiles; ++nt) sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.f;
#pragma unroll
            for (int np = 0; np < kTiles; ++np) {
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4(sK + swz(np * 16 + (lane & 7) + ((lane >> 4) << 3), 2 * ks + ((lane >> 3) & 1), 8), b0, b1,
                            b2, b3);
                    mma_m16n8k16(sacc[2 * np], qa[ks], b0, b1);
                    mma_m16n8k16(sacc[2 * np + 1], qa[ks], b2, b3);
                }
            }
            // ---- exact softmax over the T keys of rows g and g + 8 (a row lives in the 4 lanes of a quad)
            float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < 2 * kTiles; ++nt) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const bool key_ok = (8 * nt + 2 * t4 + i) < T;
                    sacc[nt][i] = key_ok ? sacc[nt][i] * scale_log2 : -INFINITY;
                    sacc[nt][2 + i] = key_ok ? sacc[nt][2 + i] * scale_log2 : -INFINITY;
                    m0 = fmaxf(m0, sacc[nt][i]);
                    m1 = fmaxf(m1, sacc[nt][2 + i]);
                }
            }
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            float l0 = 0.f, l1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 2 * kTiles; ++nt) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    sacc[nt][i] = exp2f(sacc[nt][i] - m0);
                    sacc[nt][2 + i] = exp2f(sacc[nt][2 + i] - m1);
                    l0 += sacc[nt][i];
                    l1 += sacc[nt][2 + i];
                }
            }
            l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
            l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
            const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
            // P = hi + lo, both fp16 (at most 64 keys per query: the fp16 rounding of P is not averaged away)
            uint32_t pa[kTiles][4], pl[kTiles][4];
#pragma unroll
            for (int kb = 0; kb < kTiles; ++kb) {
                split_h2(sacc[2 * kb][0] * inv0, sacc[2 * kb][1] * inv0, pa[kb][0], pl[kb][0]);
                split_h2(sacc[2 * kb][2] * inv1, sacc[2 * kb][3] * inv1, pa[kb][1], pl[kb][1]);
                split_h2(sacc[2 * kb + 1][0] * inv0, sacc[2 * kb + 1][1] * inv0, pa[kb][2], pl[kb][2]);
                split_h2(sacc[2 * kb + 1][2] * inv1, sacc[2 * kb + 1][3] * inv1, pa[kb][3], pl[kb][3]);
            }
            if (mt == 0) {
                cp_async_wait<0>();   // V has landed
                __syncwarp();
            }
            // ---- O = P V, V fragments by ldmatrix.trans (two 8-wide d tiles per instruction)
            __half* o0p = out + ((b * T + q0) * P + pix) * ldo + h * 64;
            __half* o1p = out + ((b * T + q1) * P + pix) * ldo + h * 64;
#pragma unroll
            for (int nd = 0; nd < 8; nd += 2) {
                float oa[4] = {0.f, 0.f, 0.f, 0.f}, ob[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int kb = 0; kb < kTiles; ++kb) {
                    // lane i supplies the row address of matrix i/8: (k 0-7, nd), (k 8-15, nd), (k 0-7, nd+1), (k 8-15, nd+1)
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4_t(sV + swz(16 * kb + (lane & 7) + ((lane >> 3) & 1) * 8, nd + (lane >> 4), 8), b0, b1, b2,
                              b3);
                    mma_m16n8k16(oa, pl[kb], b0, b1);
                    mma_m16n8k16(ob, pl[kb], b2, b3);
                    mma_m16n8k16(oa, pa[kb], b0, b1);
                    mma_m16n8k16(ob, pa[kb], b2, b3);
                }
                if (r0) {
                    *reinterpret_cast<uint32_t*>(o0p + 8 * nd + 2 * t4) = pack_h2(oa[0], oa[1]);
                    *reinterpret_cast<uint32_t*>(o0p + 8 * (nd + 1) + 2 * t4) = pack_h2(ob[0], ob[1]);
                }
                if (r1) {
                    *reinterpret_cast<uint32_t*>(o1p + 8 * nd + 2 * t4) = pack_h2(oa[2], oa[3]);
                    *reinterpret_cast<uint32_t*>(o1p + 8 * (nd + 1) + 2 * t4) = pack_h2(ob[2], ob[3]);
                }
            }
        }
        __syncwarp();   // the smem K / V tiles are reused by the next item
    }
}

// ===================================================================================== row softmax (in place)
__global__ void softmax_rows_kernel(__half* __restrict__ s, long long lds, int rows, int cols, float scale_log2) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int row = blockIdx.x;
    if (row >= rows) return;
    __half* r = s + (long long)row * lds;
    __shared__ float red[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    // the maximum of the scaled scores: exp2(x * scale - m) <= 1 for either sign of the scale
    float m = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, __half2float(r[c]) * scale_log2);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) red[warp] = m;
    __syncthreads();
    m = red[0];
    for (int w = 1; w < nw; ++w) m = fmaxf(m, red[w]);
    __syncthreads();
    float l = 0.f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) l += exp2f(__half2float(r[c]) * scale_log2 - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    if (lane == 0) red[warp] = l;
    __syncthreads();
    l = 0.f;
    for (int w = 0; w < nw; ++w) l += red[w];
    const float inv = 1.0f / l;
    for (int c = threadIdx.x; c < cols; c += blockDim.x)
        r[c] = __float2half_rn(exp2f(__half2float(r[c]) * scale_log2 - m) * inv);
}

}  // namespace

using namespace tc_host;

template <int kDV, bool kTwoSeg, bool kCausal = false>
static int launch_flash_kernel(const FaParams& p, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        int rc = check_cuda(cudaFuncSetAttribute(flash_attn_kernel<kDV, kTwoSeg, kCausal>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 227 * 1024),
                            "cudaFuncSetAttribute(flash_attn_kernel)");
        if (rc) return rc;
        attr_set = true;
    }
    tc_host::launch(flash_attn_kernel<kDV, kTwoSeg, kCausal>, grid, dim3(kFaThreads), smem_bytes, stream, 1, p);
    return TC_OK;
}

// split_p: P as fp16 hi + lo parts for the PV product when few keys average its rounding (cross attention: 77 + 16 keys);
// with the causal mask query i sees min(i + 1, Lk) keys, so no row sees more than Lq
static int launch_flash(const FaParams& p0, int batches, int Lk_max, bool causal, cudaStream_t stream) {
    FaParams p = p0;
    p.split_p = (causal && p.Lq < Lk_max ? p.Lq : Lk_max) <= 512 ? 1 : 0;
    // Q and K tiles of D halfs per row, V tile of DV halfs per row (80-wide rows padded to 11 chunks, tile_off)
    const size_t smem_bytes = (size_t)(tile_bytes(kFaRows, p.D) + tile_bytes(kFaKeys, p.D) + tile_bytes(kFaKeys, p.DV)) + 128;
    dim3 grid((p.Lq + kFaRows - 1) / kFaRows, p.heads * p.nv, batches);
    int rc;
    if (p.D == 80)                                                              // tc_attention only: DV = D = 80
        rc = causal ? launch_flash_kernel<80, false, true>(p, grid, smem_bytes, stream)
                    : launch_flash_kernel<80, false, false>(p, grid, smem_bytes, stream);
    else if (causal)                                                            // tc_attention only: DV = D = 64
        rc = launch_flash_kernel<64, false, true>(p, grid, smem_bytes, stream);
    else if (p.n_seg == 2)
        rc = launch_flash_kernel<64, true>(p, grid, smem_bytes, stream);        // tc_attention only: DV = D = 64
    else if (p.DV == 64)
        rc = launch_flash_kernel<64, false>(p, grid, smem_bytes, stream);
    else if (p.DV == 128)
        rc = launch_flash_kernel<128, false>(p, grid, smem_bytes, stream);
    else
        rc = launch_flash_kernel<256, false>(p, grid, smem_bytes, stream);
    if (rc) return rc;
    count_launch();
    TC_CHECK_LAUNCH("flash_attn_kernel");
    return TC_OK;
}

extern "C" int tc_attention(const TcAttention* d, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(d && d->q && d->out, "tc_attention: null pointer");
    TC_CHECK_ARG(d->n_seg == 1 || d->n_seg == 2, "tc_attention: n_seg must be 1 or 2");
    TC_CHECK_ARG(d->q_batches > 0 && d->Lq > 0 && d->heads > 0, "tc_attention: empty problem");
    TC_CHECK_ARG(d->ldq % 8 == 0 && d->ldo % 8 == 0, "tc_attention: strides must be multiples of 8");
    TC_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->q) | reinterpret_cast<uintptr_t>(d->out)) & 15) == 0,
                 "tc_attention: operands must be 16-byte aligned");
    TC_CHECK_ARG(d->head_dim == 0 || d->head_dim == 64 || d->head_dim == 80, "tc_attention: head_dim must be 0, 64 or 80");
    TC_CHECK_ARG(d->causal == 0 || d->causal == 1, "tc_attention: causal must be 0 or 1");
    const int D = d->head_dim == 80 ? 80 : 64;
    TC_CHECK_ARG(d->n_seg == 1 || (D == 64 && !d->causal),
                 "tc_attention: head dim 80 and causal masking take one key/value segment");
    FaParams p;
    memset(&p, 0, sizeof(p));
    int Lk_max = 0;
    for (int s = 0; s < d->n_seg; ++s) {
        TC_CHECK_ARG(d->k[s] && d->v[s] && d->Lk[s] > 0 && d->kv_div[s] > 0, "tc_attention: bad kv segment");
        TC_CHECK_ARG(d->ldk[s] % 8 == 0 && d->ldv[s] % 8 == 0, "tc_attention: kv strides must be multiples of 8");
        TC_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->k[s]) | reinterpret_cast<uintptr_t>(d->v[s])) & 15) == 0,
                     "tc_attention: operands must be 16-byte aligned");
        p.seg[s].k = reinterpret_cast<const __half*>(d->k[s]);
        p.seg[s].v = reinterpret_cast<const __half*>(d->v[s]);
        p.seg[s].ldk = d->ldk[s];
        p.seg[s].ldv = d->ldv[s];
        p.seg[s].Lk = d->Lk[s];
        p.seg[s].kv_div = d->kv_div[s];
        Lk_max = d->Lk[s] > Lk_max ? d->Lk[s] : Lk_max;
    }
    p.q = reinterpret_cast<const __half*>(d->q);
    p.ldq = d->ldq;
    p.Lq = d->Lq;
    p.heads = d->heads;
    p.D = D;
    p.DV = D;
    p.nv = 1;
    p.n_seg = d->n_seg;
    p.out = reinterpret_cast<__half*>(d->out);
    p.ldo = d->ldo;
    p.scale_log2 = d->scale * 1.4426950408889634f;
    return launch_flash(p, d->q_batches, Lk_max, d->causal != 0, stream);
}

extern "C" int tc_attention_wide(const void* q, const void* k, const void* v, long long ldq, long long ldk, long long ldv,
                                 void* out, long long ldo, int batches, int Lq, int Lk, int D, float scale, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(q && k && v && out, "tc_attention_wide: null pointer");
    TC_CHECK_ARG(batches > 0 && Lq > 0 && Lk > 0, "tc_attention_wide: empty problem");
    TC_CHECK_ARG(D >= 64 && D <= 512 && D % 64 == 0 && (D <= 256 || D % 128 == 0),
                 "tc_attention_wide: head dim must be a multiple of 64 (of 128 above 256), at most 512");
    TC_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "tc_attention_wide: strides must be multiples of 8");
    TC_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                   reinterpret_cast<uintptr_t>(out)) & 15) == 0, "tc_attention_wide: operands must be 16-byte aligned");
    FaParams p;
    memset(&p, 0, sizeof(p));
    p.q = reinterpret_cast<const __half*>(q);
    p.ldq = ldq;
    p.Lq = Lq;
    p.heads = 1;
    p.D = D;
    // value columns per CTA: the widest chunk that divides D (each CTA recomputes Q K^T, so fewer chunks = fewer flops;
    // D = 192 takes three 64-column chunks)
    p.DV = D % 256 == 0 ? 256 : (D % 128 == 0 ? 128 : 64);
    p.nv = D / p.DV;
    TC_CHECK_ARG(p.nv * p.DV == D, "tc_attention_wide: value chunk does not divide the head dim");
    p.n_seg = 1;
    p.seg[0].k = reinterpret_cast<const __half*>(k);
    p.seg[0].v = reinterpret_cast<const __half*>(v);
    p.seg[0].ldk = ldk;
    p.seg[0].ldv = ldv;
    p.seg[0].Lk = Lk;
    p.seg[0].kv_div = 1;
    p.out = reinterpret_cast<__half*>(out);
    p.ldo = ldo;
    p.scale_log2 = scale * 1.4426950408889634f;
    return launch_flash(p, batches, Lk, false, stream);
}

extern "C" int tc_debug_read_attn_trace(unsigned long long* host_dst, int count) {
    (void)host_dst;
    (void)count;
    return fail(TC_ERR_INVALID, "tc_debug_read_attn_trace: the attention kernel records no timeline");
}

// 16 < T <= 64: kTiles = ceil(T / 16); 4 warps x (K + V) tiles of 16 kTiles rows x 128 bytes (up to 64 KiB)
template <int kTiles>
static int launch_temporal64(dim3 grid, cudaStream_t stream, const __half* q, const __half* k, const __half* v,
                             long long ld, __half* out, long long ldo, int B, int T, int P, int heads, float sl2) {
    constexpr int smem_bytes = 4 * 2 * kTiles * 16 * 128;
    static bool attr_set = false;
    if (!attr_set) {
        int rc = check_cuda(cudaFuncSetAttribute(temporal_attn_mma64_kernel<kTiles>,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes),
                            "cudaFuncSetAttribute(temporal_attn_mma64_kernel)");
        if (rc) return rc;
        attr_set = true;
    }
    tc_host::launch(temporal_attn_mma64_kernel<kTiles>, grid, dim3(128), smem_bytes, stream, 1, q, k, v, ld, out, ldo, B,
                    T, P, heads, sl2);
    return TC_OK;
}

extern "C" int tc_temporal_attention(const void* q, const void* k, const void* v, long long ld, void* out,
                                     long long ldo, int B, int T, int P, int heads, float scale, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(q && k && v && out, "tc_temporal_attention: null pointer");
    TC_CHECK_ARG(B > 0 && T > 0 && T <= 64 && P > 0 && heads > 0, "tc_temporal_attention: need 0 < T <= 64");
    TC_CHECK_ARG(ld % 8 == 0 && ldo % 8 == 0, "tc_temporal_attention: strides must be multiples of 8");
    TC_CHECK_ARG(ld >= 64LL * heads && ldo >= 64LL * heads, "tc_temporal_attention: ld and ldo must be at least heads * 64");
    TC_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                   reinterpret_cast<uintptr_t>(out)) & 15) == 0, "tc_temporal_attention: operands must be 16-byte aligned");
    const long long items = (long long)B * P * heads;
    const float sl2 = scale * 1.4426950408889634f;
    const __half* qp = reinterpret_cast<const __half*>(q);
    const __half* kp = reinterpret_cast<const __half*>(k);
    const __half* vp = reinterpret_cast<const __half*>(v);
    __half* op = reinterpret_cast<__half*>(out);
    long long blocks = (items + 3) / 4;
    const long long cap = 16LL * sm_count();
    if (blocks > cap) blocks = cap;
    int rc = TC_OK;
    if (T <= 16)
        tc_host::launch(temporal_attn_mma_kernel, dim3((unsigned)blocks), dim3(128), 0, stream, 1, qp, kp, vp, ld, op, ldo, B, T, P, heads, sl2);
    else if (T <= 32)
        rc = launch_temporal64<2>(dim3((unsigned)blocks), stream, qp, kp, vp, ld, op, ldo, B, T, P, heads, sl2);
    else if (T <= 48)
        rc = launch_temporal64<3>(dim3((unsigned)blocks), stream, qp, kp, vp, ld, op, ldo, B, T, P, heads, sl2);
    else
        rc = launch_temporal64<4>(dim3((unsigned)blocks), stream, qp, kp, vp, ld, op, ldo, B, T, P, heads, sl2);
    if (rc) return rc;
    count_launch();
    TC_CHECK_LAUNCH("temporal_attn_kernel");
    return TC_OK;
}

extern "C" int tc_softmax_rows(void* s, long long lds, int rows, int cols, float scale, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(s && rows > 0 && cols > 0, "tc_softmax_rows: bad arguments");
    TC_CHECK_ARG(lds >= cols, "tc_softmax_rows: lds must be at least cols");
    tc_host::launch(softmax_rows_kernel, dim3(rows), dim3(256), 0, stream, 1, reinterpret_cast<__half*>(s), lds, rows, cols,
                                                  scale * 1.4426950408889634f);
    count_launch();
    TC_CHECK_LAUNCH("softmax_rows_kernel");
    return TC_OK;
}
