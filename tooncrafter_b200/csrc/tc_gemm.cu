// tooncrafter_b200 — implicit-GEMM convolution / linear layer on wgmma (sm_90a).
//
// One warp-specialised kernel serves every dense contraction of the UNet and the VAE decoder (reference call sites
// listed in include/tooncrafter_b200.h).  One CTA computes one 128 x BN output tile (or one k-slice of it):
//
//   warpgroup 0    TMA producer  : one elected thread; per k-block one 4-D box of the channels-last activation (im2col
//                                  by coordinate offset; out-of-bounds rows/cols are zero-filled by TMA == padding) and
//                                  one 2-D box of the [Cout][taps*C] weight matrix, both 128B-swizzled, into a ring of
//                                  `stages` shared-memory slots guarded by full / empty mbarriers.  Before the first
//                                  k-block it issues the tile's residual (32-column boxes, 64B-swizzled) into a region
//                                  of its own, on an mbarrier of its own, so the residual lands during the k-loop.
//                  warps 1-3     : during the k-loop, per-row LayerNorm statistics (partial slots summed) and the bias2
//                                  rows the tile spans, into shared memory (named barrier 2).  The epilogue therefore
//                                  reads no global memory, and its stores do not wait behind its loads.
//   warpgroups 1-2 wgmma         : each owns 64 of the tile's 128 rows; one m64nNk16 instruction per k16 step with
//                                  N = BNp (BN rounded up to 32), so A is read from shared memory once per step for all
//                                  columns; fp32 accumulators in registers, one k-block in flight behind the one being
//                                  issued.  The k-loop makes no function call (see tc::mbar_wait), which would make
//                                  ptxas serialise the wgmmas.  After the last k-block the same 256 threads run the
//                                  epilogue on the accumulator registers, in their fragment layout: folded LayerNorm /
//                                  bias / timestep embedding / scale / residual (ldmatrix from its boxes) or GEGLU ->
//                                  fp16 -> stmatrix into an output tile in the drained operand ring, laid out as the
//                                  swizzled boxes of an output tensor map -> TMA stores, which clip the rows and columns
//                                  past the output extent (TMA writes whole 16-byte chunks, so the last n % 8 columns
//                                  of an n-column output are stored by one thread per row).  Optional per-row {sum, sumsq} of the stored fp16 outputs
//                                  (for the consumer's LayerNorm fold) are read back from that tile, one row per thread.
//   split-K (few output tiles, long K loops): every slice parks its fp32 accumulators in a workspace, takes a ticket,
//   and the last slice to arrive sums all slices in slice order (deterministic) into its registers and runs the
//   epilogue.
//
// Algorithmic flops = 2 * M * n_cols * taps * C.
#include <stdlib.h>

#include "tc_common.cuh"
#include "tc_host.h"

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                          // 64 halfs = one 128-byte swizzle row
constexpr int kAStageBytes = kBlockM * kBlockK * 2;  // 16 KiB
constexpr int kThreads = 384;                        // warpgroup 0 TMA, warpgroups 1-2 MMA + epilogue
constexpr int kEpiThreads = 256;

constexpr int kResBoxCols = 32;                      // residual box: 32 halfs = one 64-byte swizzle row
constexpr int kResBoxBytes = kBlockM * kResBoxCols * 2;   // 8 KiB region per residual box

struct alignas(64) GemmKParams {
    CUtensorMap tmA;
    CUtensorMap tmB;
    CUtensorMap tmR;                // residual [oN][oH][oW][n_cols] (row stride ldr), boxes of 32 columns
    CUtensorMap tmO;                // output [oN][oH][oW][out_tma_cols] (row stride ldc), boxes of 2^out_box_lg columns
    int out_box_lg;                 // 5: 32-column boxes, 64B-swizzled; 4: 16-column boxes, 32B-swizzled
    int out_tma_cols;               // output columns stored by TMA: out_cols rounded down to 8 (0: no output map)
    int out_cols;                   // output columns (GEGLU: n_cols / 2); the last out_cols % 8 are stored by threads
    int res_boxes;                  // residual boxes per tile (ceil(BN / 32)), 0 without a residual
    uint32_t res_bytes;             // residual bytes delivered per tile
    uint32_t res_smem;              // shared-memory region of the residual boxes (res_boxes x 8 KiB)
    uint32_t b2_smem;               // shared-memory region of the staged bias2 rows (slots x BN halfs)
    int b2_per_row;                 // 1: one bias2 slot per tile row (a tile spans more bias2 rows than it has rows);
                                    // 0: one slot per bias2 row the tile spans, from its first output row's
    int taps;
    int tap_dx[TC_MAX_TAPS], tap_dy[TC_MAX_TAPS], tap_dn[TC_MAX_TAPS];
    int kc_per_tap;
    int TW, TH, TN;
    int oW, oH, oN;
    int tiles_x, tiles_y;           // spatial tiling of the M dimension
    int tiles_nn;                   // tiles along N
    int BN;                         // output columns per tile (GEGLU: value + gate columns)
    int ksplit, kb_per;             // k-slices per tile, k-blocks per slice
    float* ws_partial;              // [tiles][ksplit][128 rows][BNp] floats
    unsigned int* ws_ticket;        // [tiles], zero between launches (the last slice resets it)
    int n_cols;
    int stages;
    uint32_t a_bytes;               // bytes delivered per A box
    uint32_t b_bytes;               // bytes delivered per B box (BNp rows of 128 bytes)
    uint32_t ring_bytes;            // operand ring (reused as the fp16 output tile)
    __half* out;
    long long ldc;
    const float* bias;
    const __half* bias2;
    long long bias2_ld;
    int bias2_rows_per;
    float acc_scale;
    int geglu;
    const float2* ln_stats;  // per output row {mean, rstd} (ln_nslots == 0) or [M][ln_nslots] partial {sum, sumsq}
    const float* ln_u;       // per column sum_k Wt[j][k]
    int ln_nslots;
    float ln_eps, ln_inv_c;
    float2* row_stats;       // producer: per-row {sum, sumsq} partials, [M][row_stats_slots]
    int row_stats_slots;
};

__device__ __forceinline__ uint32_t pack_h2(float x, float y) {
    __half2 h = __floats2half2_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&h);
}

// output row m of tile row `row` (rows in the box's (TW, TH, TN) order, x fastest); false past the output extent
__device__ __forceinline__ bool tile_row(const GemmKParams& p, int tx, int ty, int tn, int row, long long& m) {
    const int rx = row % p.TW;
    const int ry = (row / p.TW) % p.TH;
    const int rn = row / (p.TW * p.TH);
    const int x = tx * p.TW + rx, y = ty * p.TH + ry, n = tn * p.TN + rn;
    m = ((long long)n * p.oH + y) * p.oW + x;
    return (rn < p.TN) && (x < p.oW) && (y < p.oH) && (n < p.oN);
}

// bias2 row of the tile's first output row
__device__ __forceinline__ long long tile_bias2_first(const GemmKParams& p, int tx, int ty, int tn) {
    const long long m0 = ((long long)tn * p.TN * p.oH + ty * p.TH) * p.oW + tx * p.TW;
    return m0 / p.bias2_rows_per;
}

// Byte offset of 16-byte chunk `chunk` (tile columns 8 chunk .. 8 chunk + 7) of tile row `row` in a tile held as TMA
// boxes of 2^lg columns (lg = 4 or 5), each [128 rows][2^(lg+1) bytes] with the swizzle of that row width (32B or 64B):
// chunk q of a row sits at q ^ (bits 7.. of the row's offset).  The eight rows of one 8x8 ldmatrix / stmatrix matrix then
// fall on eight different 16-byte bank groups.
__device__ __forceinline__ uint32_t swz_offset(int lg, int row, int chunk) {
    const int per_row = 1 << (lg - 3);
    const uint32_t row_off = (uint32_t)row << (lg + 1);
    const uint32_t q = (uint32_t)(chunk & (per_row - 1)) ^ ((row_off >> 7) & (uint32_t)(per_row - 1));
    return (uint32_t)(chunk >> (lg - 3)) * (uint32_t)(kBlockM << (lg + 1)) + row_off + (q << 4);
}

// four 8x8 fp16 matrices; lanes 8 i .. 8 i + 7 give the row addresses of matrix i, register i holds this lane's pair
// (row lane / 4, columns 2 (lane % 4) + {0, 1}) of matrix i: the wgmma accumulator fragment order
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr)
                 : "memory");
}
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]),
                 "r"(r[2]), "r"(r[3])
                 : "memory");
}

__device__ __forceinline__ float2 h2_to_f2(uint32_t u) {
    return __half22float2(*reinterpret_cast<const __half2*>(&u));
}

// kNJ = BNp / 32 (BNp = BN rounded up to 32): the wgmma is m64n(32 kNJ)k16
template <int kNJ>
__global__ void __launch_bounds__(kThreads, 1) tc_gemm_kernel(const __grid_constant__ GemmKParams p) {
    tc::pdl_launch_dependents();   // the successor's prologue may overlap this kernel; it blocks in its own pdl_wait
    constexpr int kBNp = kNJ * 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

    const int S = p.stages;
    const int BN = p.BN;
    uint8_t* sA = smem;
    uint8_t* sB = smem + (size_t)S * kAStageBytes;
    uint8_t* s_out = smem;                         // fp16 output tile (TMA store boxes), after the ring has drained
    uint8_t* s_res = smem + p.ring_bytes;          // residual boxes: [res_boxes][128 rows][64 B], 64B-swizzled
    __half* s_b2 = reinterpret_cast<__half*>(s_res + p.res_smem);   // [bias2_rows_max][BN]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_res + p.res_smem + p.b2_smem);
    uint64_t* empty_bar = full_bar + S;
    uint64_t* res_bar = empty_bar + S;
    float* s_bias = reinterpret_cast<float*>(res_bar + 1);     // [256]
    float* s_u = s_bias + 256;                                 // [256]
    float2* s_rs = reinterpret_cast<float2*>(s_u + 256);       // [128] row statistics of column group 1
    float2* s_ln = s_rs + 128;                                 // [128] per-row LayerNorm {mean, rstd}
    int* s_flag = reinterpret_cast<int*>(s_ln + 128);

    const int tid = threadIdx.x;
    if (tid == 0) {
        tc::tma_prefetch_desc(&p.tmA);
        tc::tma_prefetch_desc(&p.tmB);
        if (p.out_tma_cols) tc::tma_prefetch_desc(&p.tmO);
        if (p.res_boxes) tc::tma_prefetch_desc(&p.tmR);
        for (int s = 0; s < S; ++s) {
            tc::mbar_init(&full_bar[s], 1);
            tc::mbar_init(&empty_bar[s], 8);   // one arrival per consumer warp
        }
        tc::mbar_init(res_bar, 1);
        tc::fence_mbar_init();
    }
    __syncthreads();
    tc::pdl_wait();

    // work item -> (tile, k-slice); tile -> (N tile fastest, M tile): CTAs that run side by side share rows of A
    const int wi = (int)blockIdx.x;
    const int tile = wi / p.ksplit;
    const int ks = wi - tile * p.ksplit;
    const int nt = tile % p.tiles_nn;
    const int mt = tile / p.tiles_nn;
    const int tx = mt % p.tiles_x;
    const int ty = (mt / p.tiles_x) % p.tiles_y;
    const int tn = mt / (p.tiles_x * p.tiles_y);
    const int main_kblocks = p.taps * p.kc_per_tap;
    const int kb_begin = ks * p.kb_per;
    const int kb_end = min(kb_begin + p.kb_per, main_kblocks);

    if (tid >= 32 && tid < 128) {
        // ------------------------------------------------------------------ warps 1-3: epilogue operands, during the k-loop
        // per-row LayerNorm statistics (partial slots summed in slot order, as a fixed order keeps results deterministic)
        // and the bias2 rows of the tile; the MMA warpgroups wait for them (named barrier 2) only after their k-loop
        const int pt = tid - 32;
        if (p.ln_stats) {
            for (int row = pt; row < kBlockM; row += 96) {
                long long m;
                float mean = 0.f, rstd = 1.f;
                if (tile_row(p, tx, ty, tn, row, m)) {
                    if (p.ln_nslots > 0) {
                        float s1 = 0.f, s2 = 0.f;
                        const float2* ps = p.ln_stats + m * p.ln_nslots;
                        for (int i = 0; i < p.ln_nslots; ++i) {
                            const float2 st = __ldg(ps + i);
                            s1 += st.x;
                            s2 += st.y;
                        }
                        mean = s1 * p.ln_inv_c;
                        rstd = rsqrtf(fmaxf(s2 * p.ln_inv_c - mean * mean, 0.f) + p.ln_eps);
                    } else {
                        const float2 st = __ldg(p.ln_stats + m);
                        mean = st.x;
                        rstd = st.y;
                    }
                }
                s_ln[row] = make_float2(mean, rstd);
            }
        }
        if (p.bias2) {
            // slots: bias2 rows [first, last] of the tile's first and last output rows (a tile may straddle sample
            // boundaries), or the bias2 row of each tile row (b2_per_row); columns past n_cols are zero (they feed no
            // stored output)
            long long m_last;
            const int xl = min(p.TW, p.oW - tx * p.TW) - 1, yl = min(p.TH, p.oH - ty * p.TH) - 1;
            const int nl = min(p.TN, p.oN - tn * p.TN) - 1;
            tile_row(p, tx, ty, tn, (nl * p.TH + yl) * p.TW + xl, m_last);
            const long long first = tile_bias2_first(p, tx, ty, tn);
            const int slots = p.b2_per_row ? kBlockM : (int)(m_last / p.bias2_rows_per - first) + 1;
            const int chunks = BN / 8;
            for (int i = pt; i < slots * chunks; i += 96) {
                const int r = i / chunks, c = 8 * (i - r * chunks);
                const int col = nt * BN + c;
                long long b2r = first + r;
                if (p.b2_per_row) {
                    long long m;
                    if (!tile_row(p, tx, ty, tn, r, m)) continue;
                    b2r = m / p.bias2_rows_per;
                }
                const __half* src = p.bias2 + b2r * p.bias2_ld + col;
                __half* dst = s_b2 + r * BN + c;
                if (col + 8 <= p.n_cols) {
                    *reinterpret_cast<uint4*>(dst) = __ldg(reinterpret_cast<const uint4*>(src));
                } else {
                    for (int j = 0; j < 8; ++j) dst[j] = col + j < p.n_cols ? src[j] : __float2half_rn(0.f);
                }
            }
        }
        asm volatile("bar.arrive 2, 352;" ::: "memory");
        return;
    }
    if (tid < 32) {
        // ------------------------------------------------------------------ TMA producer
        if (tc::elect_one()) {
            const int x0 = tx * p.TW, y0 = ty * p.TH, n0 = tn * p.TN;
            if (p.res_boxes) {
                // the residual tile lands during the k-loop, on an mbarrier of its own.  Under split-K every slice loads
                // it: which slice runs the epilogue is known only from its ticket, after its k-loop, and one more
                // 128 x BN fp16 read is small next to a slice's operand traffic (>= 8 k-blocks of A and B)
                tc::mbar_arrive_expect_tx(res_bar, p.res_bytes);
                for (int b = 0; b < p.res_boxes; ++b)
                    tc::tma_load_4d(s_res + b * kResBoxBytes, &p.tmR, res_bar, nt * BN + b * kResBoxCols, x0, y0, n0);
            }
            int stage = 0;
            uint32_t phase = 0;
            int tap = kb_begin / p.kc_per_tap;
            int kc = kb_begin - tap * p.kc_per_tap;
            for (int kb = kb_begin; kb < kb_end; ++kb) {
                tc::mbar_wait(&empty_bar[stage], phase ^ 1u);
                tc::mbar_arrive_expect_tx(&full_bar[stage], p.a_bytes + p.b_bytes);
                tc::tma_load_4d(sA + (size_t)stage * kAStageBytes, &p.tmA, &full_bar[stage], kc * kBlockK,
                                x0 + p.tap_dx[tap], y0 + p.tap_dy[tap], n0 + p.tap_dn[tap]);
                tc::tma_load_2d(sB + (size_t)stage * p.b_bytes, &p.tmB, &full_bar[stage], kb * kBlockK, nt * BN);
                if (++kc == p.kc_per_tap) { kc = 0; ++tap; }
                if (++stage == S) { stage = 0; phase ^= 1u; }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- MMA warpgroups
    const int et = tid - 128;                 // 0..255
    const int wg = et >> 7;                   // rows [64 wg, 64 wg + 64)
    const int warp = (et >> 5) & 3, lane = et & 31;
    {
        // per-column vectors of this N tile (zeros when the launch has none): the epilogue runs one branch-free form
        const int col = nt * BN + et;
        const bool ok = et < BN && col < p.n_cols;
        s_bias[et] = (ok && p.bias) ? __ldg(p.bias + col) : 0.f;
        s_u[et] = (ok && p.ln_u) ? __ldg(p.ln_u + col) : 0.f;
    }
    float acc[16 * kNJ];   // element 16 j + i: column 32 j + 8 (i >> 2) + 2 (lane % 4) + (i & 1)
#pragma unroll
    for (int i = 0; i < 16 * kNJ; ++i) acc[i] = 0.f;
    {
        const uint64_t a_desc0 = tc::wgmma_desc_sw128(tc::smem_u32(sA + wg * 64 * 128));
        const uint64_t b_desc0 = tc::wgmma_desc_sw128(tc::smem_u32(sB));
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int kb = kb_begin; kb < kb_end; ++kb) {
            tc::mbar_wait(&full_bar[stage], phase);
            tc::wgmma_fence();
            const uint64_t ad = a_desc0 + (uint64_t)(stage * (kAStageBytes >> 4));
            const uint64_t bd = b_desc0 + (uint64_t)(stage * (p.b_bytes >> 4));
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k)   // +32 bytes along the swizzled K row per k16 step
                tc::wgmma_m64nNk16<kNJ>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k));
            tc::wgmma_commit();
            tc::wgmma_wait<1>();              // the previous k-block's MMAs have finished reading their slot
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
            }
            prev = stage;
            if (++stage == S) { stage = 0; phase ^= 1u; }
        }
        tc::wgmma_wait<0>();
    }
    // every MMA of both warpgroups has retired (the operand ring becomes the fp16 output tile), and warps 1-3 have
    // stored the LayerNorm statistics and bias2 rows
    asm volatile("bar.sync 2, 352;" ::: "memory");
    // every k-slice waits, so that no CTA exits with its residual load in flight
    if (p.res_boxes) tc::mbar_wait(res_bar, 0);

    if (p.ksplit > 1) {
        // park this slice's accumulators (float4 v of thread et at v * 256 + et: a warp's store writes 512 contiguous
        // bytes), take a ticket; only the last slice of the tile goes on and sums the slices in slice order into acc
        constexpr int kSliceV4 = kBlockM * kBNp / 4;   // = 4 kNJ float4 per thread
        float4* ws_tile = reinterpret_cast<float4*>(p.ws_partial) + (long long)tile * p.ksplit * kSliceV4;
        float4* wslice = ws_tile + (long long)ks * kSliceV4;
#pragma unroll
        for (int v = 0; v < 4 * kNJ; ++v)
            __stcg(wslice + v * kEpiThreads + et,
                   make_float4(acc[4 * v], acc[4 * v + 1], acc[4 * v + 2], acc[4 * v + 3]));
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (et == 0) {
            unsigned int* tk = p.ws_ticket + tile;
            const unsigned int t = atomicAdd(tk, 1u);
            const bool last = (t == (unsigned int)(p.ksplit - 1));
            if (last) *tk = 0u;                     // ready for the next launch (stream order)
            s_flag[0] = last ? 1 : 0;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (s_flag[0] == 0) return;
        __threadfence();
#pragma unroll
        for (int i = 0; i < 16 * kNJ; ++i) acc[i] = 0.f;
        for (int sl = 0; sl < p.ksplit; ++sl) {
            const float4* src = ws_tile + (long long)sl * kSliceV4 + et;
#pragma unroll
            for (int v = 0; v < 4 * kNJ; ++v) {
                const float4 u = __ldcg(src + v * kEpiThreads);
                acc[4 * v] += u.x;
                acc[4 * v + 1] += u.y;
                acc[4 * v + 2] += u.z;
                acc[4 * v + 3] += u.w;
            }
        }
    }

    // ---------------------------------------------------------------------- epilogue, in the accumulators' layout
    // Thread (warp, lane) of warpgroup wg holds rows rb and rb + 8 (rb = 64 wg + 16 warp + lane / 4).  Accumulator
    // 8 t + 2 k + e is row rb + 8 (k & 1), column 16 t + 8 (k >> 1) + 2 (lane % 4) + e: per 16-column group t, its four
    // register pairs are this lane's parts of the four 8x8 matrices (k & 1, k >> 1) of one ldmatrix / stmatrix .x4.
    const bool geglu = p.geglu != 0;
    const int width = geglu ? (BN >> 1) : BN;                   // output columns per tile
    const int col0 = nt * width;                                // first output column of the tile
    const int lg = p.out_box_lg;
    const int rb = wg * 64 + warp * 16 + (lane >> 2);
    const int cl = 2 * (lane & 3);
    // row and 16-byte column chunk (within the group) this lane addresses for ldmatrix / stmatrix: matrix lane / 8
    const int mrow = wg * 64 + warp * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
    const int mchunk = lane >> 4;
    float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
    const __half* b2row[2] = {s_b2, s_b2};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = rb + 8 * h;
        if (p.ln_stats) {
            const float2 st = s_ln[r];
            mean[h] = st.x;
            rstd[h] = st.y;
        }
        long long m;
        if (p.bias2 && tile_row(p, tx, ty, tn, r, m))   // rows past the output extent are computed but not stored
            b2row[h] = s_b2 + (p.b2_per_row ? r : m / p.bias2_rows_per - tile_bias2_first(p, tx, ty, tn)) * BN;
    }
    // the tile row this thread reads back once the stores are issued (partial last chunk, row statistics)
    const int row = et & 127;
    long long m;
    const bool row_ok = tile_row(p, tx, ty, tn, row, m);
    const uint32_t out_u32 = tc::smem_u32(s_out), res_u32 = tc::smem_u32(s_res);
    if (!geglu) {
#pragma unroll
        for (int t = 0; t < 2 * kNJ; ++t) {
            if (16 * t >= width) break;
            uint32_t res[4];
            if (p.res_boxes) ldmatrix_x4(res_u32 + swz_offset(5, mrow, 2 * t + mchunk), res);
            uint32_t packed[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int h = k & 1, c = 16 * t + 8 * (k >> 1) + cl;
                const float2 u = *reinterpret_cast<const float2*>(s_u + c);
                const float2 b = *reinterpret_cast<const float2*>(s_bias + c);
                float v0 = rstd[h] * (acc[8 * t + 2 * k] - mean[h] * u.x) + b.x;
                float v1 = rstd[h] * (acc[8 * t + 2 * k + 1] - mean[h] * u.y) + b.y;
                if (p.bias2) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(b2row[h] + c));
                    v0 += f.x;
                    v1 += f.y;
                }
                if (p.acc_scale != 1.0f) {
                    v0 *= p.acc_scale;
                    v1 *= p.acc_scale;
                }
                if (p.res_boxes) {
                    const float2 f = h2_to_f2(res[k]);
                    v0 += f.x;
                    v1 += f.y;
                }
                packed[k] = pack_h2(v0, v1);
            }
            stmatrix_x4(out_u32 + swz_offset(lg, mrow, 2 * t + mchunk), packed);
        }
    } else {
        // weight rows of this N tile are [value half | gate half], BN = 32 kNJ: gate column c + width is accumulator
        // 8 (t + kNJ) + 2 k + e of the same thread
#pragma unroll
        for (int t = 0; t < kNJ; ++t) {
            uint32_t packed[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int h = k & 1, c = 16 * t + 8 * (k >> 1) + cl, g = c + 16 * kNJ;
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float a = rstd[h] * (acc[8 * t + 2 * k + e] - mean[h] * s_u[c + e]) + s_bias[c + e];
                    const float xg =
                        rstd[h] * (acc[8 * (t + kNJ) + 2 * k + e] - mean[h] * s_u[g + e]) + s_bias[g + e];
                    v[e] = a * tc::gelu_erf_f(xg);
                }
                packed[k] = pack_h2(v[0], v[1]);
            }
            stmatrix_x4(out_u32 + swz_offset(lg, mrow, 2 * t + mchunk), packed);
        }
    }
    // the tile leaves as TMA boxes of 2^lg columns over the output's (TW, TH, TN) box; TMA drops the rows and columns
    // past the output extent.  It writes whole 16-byte chunks, so the last out_cols % 8 columns (a partial chunk) are
    // not part of the output map: one thread per row stores them
    tc::fence_proxy_async_smem();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (et == 0 && p.out_tma_cols > col0) {
        for (int b = 0; b < (width >> lg); ++b)
            tc::tma_store_4d(s_out + b * (kBlockM << (lg + 1)), &p.tmO, col0 + (b << lg), tx * p.TW, ty * p.TH,
                             tn * p.TN);
        tc::bulk_commit_group();
    }
    {
        const int tail = p.out_tma_cols - col0;   // tile column of the partial chunk
        if (p.out_cols > p.out_tma_cols && tail >= 0 && tail < width && et >= 128) {
            if (row_ok) {
                const uint4 u = *reinterpret_cast<const uint4*>(s_out + swz_offset(lg, row, tail >> 3));
                const __half* hv = reinterpret_cast<const __half*>(&u);
                __half* dst = p.out + m * p.ldc + p.out_tma_cols;
#pragma unroll
                for (int i = 0; i < 7; ++i)
                    if (i < p.out_cols - p.out_tma_cols) dst[i] = hv[i];
            }
        }
    }
    if (p.row_stats) {
        // per-row {sum, sumsq} of the stored fp16 outputs, read back from the tile: one row per thread and two column
        // groups, summed in column order; column group 1 hands its partials to the thread of group 0 that owns the row
        const int cg = et >> 7;
        const int split = ((width / 16 + 1) / 2) * 16;          // group 0: [0, split), group 1: [split, width)
        const int c_end = cg == 0 ? split : width;
        float rs_sum = 0.f, rs_sq = 0.f;
        if (row_ok) {
            for (int c = cg == 0 ? 0 : split; c < c_end; c += 8) {
                const int nvalid = min(8, p.n_cols - (col0 + c));
                if (nvalid <= 0) break;
                const uint4 u = *reinterpret_cast<const uint4*>(s_out + swz_offset(lg, row, c >> 3));
                if (nvalid == 8) {
                    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 f = __half22float2(h2[i]);
                        rs_sum += f.x + f.y;
                        rs_sq = fmaf(f.x, f.x, fmaf(f.y, f.y, rs_sq));
                    }
                } else {
                    const __half* hv = reinterpret_cast<const __half*>(&u);
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        if (i < nvalid) {
                            const float f = __half2float(hv[i]);
                            rs_sum += f;
                            rs_sq = fmaf(f, f, rs_sq);
                        }
                    }
                }
            }
        }
        if (cg == 1) s_rs[row] = make_float2(rs_sum, rs_sq);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (cg == 0 && row_ok) {
            const float2 o = s_rs[row];
            p.row_stats[m * p.row_stats_slots + nt] = make_float2(rs_sum + o.x, rs_sq + o.y);
        }
    }
    // the stores have completed (not only read the tile) before the CTA exits: a dependent kernel's
    // griddepcontrol.wait then sees the output
    if (et == 0) tc::bulk_wait_group<0>();
}

// Tile-shape heuristic: pick (block_n, k-slices) minimising   waves x per-tile cycles   with a small model of one
// k-block (M128 x bn x K64): tensor time at the data-sheet dense fp16 rate (989 TFLOP/s over 132 SMs: ~4 bn cycles), or
// the ingest of its operands (A 16 KB + B bn x 128 B) at an assumed 52 B/clk/SM from L2, plus an assumed ~1500 cycles of
// per-tile pipeline fill / epilogue tail.  Matters for the 10x16 and 5x8 UNet levels (M = 5120 / 1280 rows), where one
// wave of 256-wide tiles leaves most SMs idle.
// Checked against per-shape sweeps of the full-width-wgmma kernel (scripts/bench_gemm.py --sweep) on the 15 largest
// shapes of a clip: 14 choices are within 5 % of the best measured (block_n, k-slices).  Known miss: the split-K term is
// too small for 5120 x 1280 at K = 11520 (3x3 conv), which splits where one 256-wide slice is ~20 % faster; a larger term
// stops 5120 x 640 at K = 5760 from splitting, which the model must keep, so a single constant cannot fit both.  The
// tensor rate, the 52 B/clk ingest and the per-tile overhead are the original estimates, not fitted.
struct TileChoice {
    int bn;
    int ksplit;
};

TileChoice choose_tiles(int tiles_m, int n_cols, int kblocks, int forced_bn, int sms, int max_ksplit, long long ws_floats) {
    const int n16 = (n_cols + 15) / 16 * 16;
    TileChoice best{n16 <= 256 ? n16 : 256, 1};
    double best_cost = 1e30;
    for (int bn = 256; bn >= 16; bn -= 16) {
        if (forced_bn > 0 && bn != forced_bn) continue;
        if (forced_bn == 0) {
            if (bn > n16) continue;
            if (n16 > 256 ? (n16 % bn != 0 || bn < 64 || bn % 32 != 0) : (bn != n16)) continue;
        }
        const int bnp = (bn + 31) / 32 * 32;
        const int tiles_n = (n_cols + bn - 1) / bn;
        const double tensor = 4.0 * bnp;
        const double ingest = (16384.0 + (double)bnp * 128.0) / 52.0;
        double kb_cycles = tensor > ingest ? tensor : ingest;
        if (kb_cycles < 200.0) kb_cycles = 200.0;
        const long long tiles = (long long)tiles_m * tiles_n;
        for (int ks = 1; ks <= max_ksplit; ++ks) {
            const int kb_per = (kblocks + ks - 1) / ks;
            if (ks > 1) {
                // slices of >= 8 k-blocks, whole-tile workspace
                if (kb_per < 8 || (kb_per * (ks - 1)) >= kblocks) continue;
                if (tiles * ks * 128 * bnp > ws_floats || tiles * 4 > TC_GEMM_WS_TICKET_BYTES) continue;
                if (bn % 32 != 0 || n_cols % bn != 0) continue;
            }
            // split-K overhead (model parameter): every slice parks 128 x bn floats in L2, a fence + ticket round trip, and
            // the last slice reads ks of them back before the usual epilogue; a 5 % margin keeps marginal cases unsplit
            const double red = ks > 1 ? 22000.0 * (bn / 256.0) * (0.5 + 0.25 * ks) : 0.0;
            const double tile_cost = (double)kb_per * kb_cycles + 1500.0 + 4.0 * bn;
            const long long waves = (tiles * ks + sms - 1) / sms;
            const double cost = ((double)waves * tile_cost + red) * (ks > 1 ? 1.05 : 1.0);
            if (cost < best_cost) {
                best_cost = cost;
                best = TileChoice{bn, ks};
            }
        }
    }
    return best;
}

using KernelFn = void (*)(GemmKParams);
const KernelFn kKernels[8] = {tc_gemm_kernel<1>, tc_gemm_kernel<2>, tc_gemm_kernel<3>, tc_gemm_kernel<4>,
                              tc_gemm_kernel<5>, tc_gemm_kernel<6>, tc_gemm_kernel<7>, tc_gemm_kernel<8>};

}  // namespace

extern "C" int tc_debug_read_gemm_trace(unsigned long long* host_dst, int count) {
    (void)host_dst;
    (void)count;
    return tc_host::fail(TC_ERR_INVALID, "tc_debug_read_gemm_trace: the GEMM kernel records no timeline");
}

static int g_last_cfg[4] = {0, 0, 0, 0};
extern "C" int tc_debug_last_gemm_config(int* out4) {
    if (!out4) return tc_host::fail(TC_ERR_INVALID, "tc_debug_last_gemm_config: null");
    for (int i = 0; i < 4; ++i) out4[i] = g_last_cfg[i];
    return TC_OK;
}

static int g_ksplit_cap = 0;   // profiling: bits 8..11 of the debug mode cap the k-slices of later launches (0 = heuristic)
extern "C" int tc_debug_set_gemm_mode(int mode) {
    g_ksplit_cap = (mode >> 8) & 15;
    return TC_OK;
}

extern "C" int tc_conv_gemm(const TcConvGemm* d, void* stream_v) {
    using namespace tc_host;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(d != nullptr, "tc_conv_gemm: null descriptor");
    TC_CHECK_ARG(d->a && d->b && d->out, "tc_conv_gemm: null operand pointer");
    TC_CHECK_ARG(d->a_C > 0 && d->a_C % kBlockK == 0, "tc_conv_gemm: C must be a positive multiple of 64");
    TC_CHECK_ARG(d->taps >= 1 && d->taps <= TC_MAX_TAPS, "tc_conv_gemm: taps out of range");
    TC_CHECK_ARG(d->oN > 0 && d->oH > 0 && d->oW > 0 && d->n_cols > 0, "tc_conv_gemm: empty problem");
    TC_CHECK_ARG((reinterpret_cast<uintptr_t>(d->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->b) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(d->out) & 15) == 0,
                 "tc_conv_gemm: operands must be 16-byte aligned");
    TC_CHECK_ARG(d->a_sW % 8 == 0 && d->a_sH % 8 == 0 && d->a_sN % 8 == 0 && d->ldb % 8 == 0 && d->ldc % 8 == 0,
                 "tc_conv_gemm: strides must be multiples of 8 elements");
    TC_CHECK_ARG((d->ln_stats == nullptr) == (d->ln_u == nullptr), "tc_conv_gemm: ln_stats and ln_u go together");
    TC_CHECK_ARG(!d->ln_stats || d->n_cols % 16 == 0, "tc_conv_gemm: folded LayerNorm needs n_cols % 16 == 0");
    TC_CHECK_ARG(!d->ln_stats || d->ln_nslots == 0 || (d->ln_nslots > 0 && d->ln_nslots <= 64 && d->taps == 1),
                 "tc_conv_gemm: partial-sum LayerNorm statistics need taps == 1 and 1..64 slots");
    TC_CHECK_ARG(!d->row_stats || (d->block_n > 0 && !(d->flags & TC_EPI_GEGLU) &&
                                   d->row_stats_slots == (d->n_cols + d->block_n - 1) / d->block_n),
                 "tc_conv_gemm: row_stats needs an explicit block_n and row_stats_slots == ceil(n_cols/block_n)");
    TC_CHECK_ARG(!d->res || (d->ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(d->res) & 15) == 0),
                 "tc_conv_gemm: residual must be 16-byte aligned");
    TC_CHECK_ARG(!d->res || d->ldr >= d->n_cols, "tc_conv_gemm: ldr must be >= n_cols");
    // bias2 rows are staged into shared memory 8 halfs (16 bytes) at a time
    TC_CHECK_ARG(!d->bias2 || (d->bias2_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(d->bias2) & 15) == 0),
                 "tc_conv_gemm: bias2 must be 16-byte aligned with bias2_ld % 8 == 0");
    TC_CHECK_ARG(d->n_cols <= d->b_rows, "tc_conv_gemm: n_cols must be <= b_rows");
    const bool geglu = (d->flags & TC_EPI_GEGLU) != 0;
    TC_CHECK_ARG(d->ldc >= (geglu ? d->n_cols / 2 : d->n_cols), "tc_conv_gemm: ldc must be >= the output width");
    int BN = d->block_n > 0 ? d->block_n : 0;   // 0: chosen below, once the M tiling is known
    TC_CHECK_ARG(BN == 0 || (BN % 16 == 0 && BN >= 16 && BN <= 256),
                 "tc_conv_gemm: block_n must be a multiple of 16 in [16,256]");
    if (geglu) {
        TC_CHECK_ARG(BN > 0 && BN % 32 == 0 && d->n_cols % BN == 0, "tc_conv_gemm: GEGLU needs n_cols % block_n == 0");
        TC_CHECK_ARG(!d->res && !d->bias2, "tc_conv_gemm: GEGLU epilogue takes bias only");
        TC_CHECK_ARG(d->acc_scale == 1.0f, "tc_conv_gemm: GEGLU epilogue takes no acc_scale");
    }

    GemmKParams p;
    memset(&p, 0, sizeof(p));
    // --- M tiling: (TW, TH, TN) box of output pixels, TW*TH*TN <= 128, minimising the tile count
    int bestTW = 1, bestTH = 1, bestTN = 1;
    long long best_tiles = -1;
    const int maxW = d->oW < kBlockM ? d->oW : kBlockM;
    for (int TW = 1; TW <= maxW; ++TW) {
        int maxH = kBlockM / TW;
        if (maxH > d->oH) maxH = d->oH;
        for (int TH = 1; TH <= maxH; ++TH) {
            int TN = kBlockM / (TW * TH);
            if (TN > d->oN) TN = d->oN;
            if (TN < 1) continue;
            // (a box may span several frames with only part of each: 10 x 16 frames tile as 16 x 2 x 4 — 40 full tiles for
            // 32 frames where whole-frame or single-frame boxes need 64 tiles of 80 rows)
            const long long tiles = (long long)((d->oW + TW - 1) / TW) * ((d->oH + TH - 1) / TH) *
                                    ((d->oN + TN - 1) / TN);
            if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && TW > bestTW) ||
                (tiles == best_tiles && TW == bestTW && TH > bestTH)) {
                best_tiles = tiles;
                bestTW = TW;
                bestTH = TH;
                bestTN = TN;
            }
        }
    }
    p.TW = bestTW;
    p.TH = bestTH;
    p.TN = bestTN;
    p.oW = d->oW;
    p.oH = d->oH;
    p.oN = d->oN;
    p.tiles_x = (d->oW + p.TW - 1) / p.TW;
    p.tiles_y = (d->oH + p.TH - 1) / p.TH;
    const int tiles_n = (d->oN + p.TN - 1) / p.TN;
    const long long tiles_m = (long long)p.tiles_x * p.tiles_y * tiles_n;
    TC_CHECK_ARG((long long)d->oN * d->oH * d->oW < (1LL << 31), "tc_conv_gemm: more than 2^31 output rows");
    // split-K only for plain epilogues (no GEGLU, no LayerNorm fold, no row statistics) with a workspace
    static const char* ksplit_env = getenv("TC_GEMM_KSPLIT");    // "1" disables, "2".."4" caps (A/B testing)
    int max_ksplit = 4;
    if (ksplit_env && ksplit_env[0] >= '1' && ksplit_env[0] <= '4') max_ksplit = ksplit_env[0] - '0';
    if (g_ksplit_cap >= 1 && g_ksplit_cap <= 4) max_ksplit = g_ksplit_cap;
    const long long ws_floats = d->workspace && d->workspace_bytes > TC_GEMM_WS_TICKET_BYTES
                                    ? (d->workspace_bytes - TC_GEMM_WS_TICKET_BYTES) / 4 : 0;
    if (geglu || d->ln_stats || d->row_stats || d->n_cols % 16 != 0 || ws_floats == 0 ||
        (reinterpret_cast<uintptr_t>(d->workspace) & 15) != 0)
        max_ksplit = 1;
    const int main_kblocks = d->taps * (d->a_C / kBlockK);
    TileChoice choice = choose_tiles((int)tiles_m, d->n_cols, main_kblocks, BN, sm_count(), max_ksplit, ws_floats);
    BN = choice.bn;
    const int BNp = (BN + 31) / 32 * 32;
    p.ksplit = choice.ksplit;
    p.kb_per = (main_kblocks + p.ksplit - 1) / p.ksplit;
    p.BN = BN;
    p.tiles_nn = (d->n_cols + BN - 1) / BN;
    p.n_cols = d->n_cols;
    p.taps = d->taps;
    for (int t = 0; t < d->taps; ++t) {
        p.tap_dx[t] = d->tap_dx[t];
        p.tap_dy[t] = d->tap_dy[t];
        p.tap_dn[t] = d->tap_dn[t];
    }
    p.kc_per_tap = d->a_C / kBlockK;
    p.a_bytes = (uint32_t)(p.TW * p.TH * p.TN) * 128u;
    p.b_bytes = (uint32_t)BNp * 128u;
    p.out = reinterpret_cast<__half*>(d->out);
    p.ldc = d->ldc;
    p.bias = d->bias;
    p.bias2 = reinterpret_cast<const __half*>(d->bias2);
    p.bias2_ld = d->bias2_ld;
    p.bias2_rows_per = d->bias2_rows_per > 0 ? d->bias2_rows_per : 1;
    p.acc_scale = d->acc_scale;
    p.geglu = geglu ? 1 : 0;
    p.ln_stats = reinterpret_cast<const float2*>(d->ln_stats);
    p.ln_u = d->ln_u;
    p.ln_nslots = d->ln_stats ? d->ln_nslots : 0;
    p.ln_eps = d->ln_eps;
    p.ln_inv_c = 1.0f / (float)d->a_C;
    p.row_stats = reinterpret_cast<float2*>(d->row_stats);
    p.row_stats_slots = d->row_stats_slots;
    p.ws_ticket = reinterpret_cast<unsigned int*>(d->workspace);
    p.ws_partial = reinterpret_cast<float*>(reinterpret_cast<char*>(d->workspace) + TC_GEMM_WS_TICKET_BYTES);

    // --- tensor maps
    {
        uint64_t dims[4] = {(uint64_t)d->a_C, (uint64_t)d->a_W, (uint64_t)d->a_H, (uint64_t)d->a_N};
        uint64_t strides[3] = {(uint64_t)d->a_sW * 2, (uint64_t)d->a_sH * 2, (uint64_t)d->a_sN * 2};
        uint32_t box[4] = {(uint32_t)kBlockK, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
        const CUtensorMap* m = get_tensor_map(d->a, 4, dims, strides, box);
        if (!m) return TC_ERR_CUDA;
        p.tmA = *m;
    }
    {
        // BNp rows per box: rows past the tile (or past b_rows, zero-filled) feed accumulator columns that are not stored
        uint64_t dims[2] = {(uint64_t)d->taps * (uint64_t)d->a_C, (uint64_t)d->b_rows};
        uint64_t strides[1] = {(uint64_t)d->ldb * 2};
        uint32_t box[2] = {(uint32_t)kBlockK, (uint32_t)BNp};
        const CUtensorMap* m = get_tensor_map(d->b, 2, dims, strides, box);
        if (!m) return TC_ERR_CUDA;
        p.tmB = *m;
    }
    if (d->res) {
        // the output tile's (TW, TH, TN) box over the residual, cut into 32-column boxes (64-byte swizzle): 32 rather
        // than 64 columns so that a 160-wide tile takes 40 KiB rather than 48 KiB, which keeps its ring at 5 stages
        uint64_t dims[4] = {(uint64_t)d->n_cols, (uint64_t)d->oW, (uint64_t)d->oH, (uint64_t)d->oN};
        uint64_t strides[3] = {(uint64_t)d->ldr * 2, (uint64_t)d->ldr * d->oW * 2, (uint64_t)d->ldr * d->oW * d->oH * 2};
        uint32_t box[4] = {(uint32_t)kResBoxCols, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
        const CUtensorMap* m = get_tensor_map(d->res, 4, dims, strides, box, 64);
        if (!m) return TC_ERR_CUDA;
        p.tmR = *m;
        p.res_boxes = (BN + kResBoxCols - 1) / kResBoxCols;
        p.res_bytes = (uint32_t)(p.res_boxes * p.TW * p.TH * p.TN * kResBoxCols * 2);
        p.res_smem = (uint32_t)(p.res_boxes * kResBoxBytes);
    }
    if (d->bias2) {
        // bias2 rows one tile can span: its output rows lie within `extent` rows of its first one.  A conv box with
        // TW < oW or TH < oH spans more than 128 consecutive output rows; past 128 bias2 rows, stage one per tile row
        const long long extent = ((long long)(p.TN - 1) * p.oH + (p.TH - 1)) * p.oW + (p.TW - 1);
        const long long span = (extent + p.bias2_rows_per - 1) / p.bias2_rows_per + 1;
        p.b2_per_row = span > kBlockM ? 1 : 0;
        p.b2_smem = (uint32_t)((p.b2_per_row ? kBlockM : span) * BN * 2);
    }

    {
        // the output tile's (TW, TH, TN) box over the output window, in boxes of 32 columns (64B swizzle), or of 16
        // (32B swizzle) when the tile width is an odd multiple of 16, so that no box reaches into the next tile's columns
        // columns past a multiple of 8 are left to the kernel's threads (a TMA store writes whole 16-byte chunks)
        const int width = geglu ? BN / 2 : BN;
        p.out_box_lg = width % 32 == 0 ? 5 : 4;
        p.out_cols = geglu ? d->n_cols / 2 : d->n_cols;
        p.out_tma_cols = p.out_cols & ~7;
        if (p.out_tma_cols > 0) {
            const uint64_t ldc = (uint64_t)d->ldc;
            uint64_t dims[4] = {(uint64_t)p.out_tma_cols, (uint64_t)d->oW, (uint64_t)d->oH, (uint64_t)d->oN};
            uint64_t strides[3] = {ldc * 2, ldc * d->oW * 2, ldc * d->oW * d->oH * 2};
            uint32_t box[4] = {1u << p.out_box_lg, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
            const CUtensorMap* m = get_tensor_map(d->out, 4, dims, strides, box, 2 << p.out_box_lg);
            if (!m) return TC_ERR_CUDA;
            p.tmO = *m;
        }
    }

    // shared memory: operand ring, residual boxes, bias2 rows, barriers, per-column vectors, per-row statistics,
    // alignment slack.  The drained ring holds the fp16 output tile (128 x BN x 2 bytes), which two stages always exceed
    const int stage_bytes = kAStageBytes + (int)p.b_bytes;
    const int kFixedSmem = 1024 + 8 * (2 * 8 + 1) + 2048 + 1024 + 1024 + 64;
    const int operand_smem = (int)(p.res_smem + p.b2_smem);
    const int smem_budget = 227 * 1024 - kFixedSmem - operand_smem;
    int stages = smem_budget / stage_bytes;
    if (stages > 8) stages = 8;
    if (stages < 2) return fail(TC_ERR_INVALID, "tc_conv_gemm: not enough shared memory for 2 stages");
    p.stages = stages;
    const int ring = stages * stage_bytes;
    p.ring_bytes = (uint32_t)ring;
    const size_t smem_bytes = (size_t)ring + operand_smem + kFixedSmem;
    TC_CHECK_ARG(smem_bytes <= 227 * 1024, "tc_conv_gemm: tile does not fit in shared memory");

    static bool attr_set = false;
    if (!attr_set) {
        for (int i = 0; i < 8; ++i) {
            int rc = check_cuda(cudaFuncSetAttribute(reinterpret_cast<const void*>(kKernels[i]),
                                                     cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024),
                                "cudaFuncSetAttribute(tc_gemm_kernel)");
            if (rc) return rc;
        }
        attr_set = true;
    }
    const long long grid = tiles_m * p.tiles_nn * p.ksplit;
    TC_CHECK_ARG(grid < (1LL << 31), "tc_conv_gemm: too many tiles");
    g_last_cfg[0] = BN, g_last_cfg[1] = 0, g_last_cfg[2] = p.ksplit, g_last_cfg[3] = stages;
    launch(kKernels[BNp / 32 - 1], dim3((unsigned)grid), dim3(kThreads), smem_bytes, stream, 1, p);
    count_launch();
    TC_CHECK_LAUNCH("tc_gemm_kernel launch");
    return TC_OK;
}
