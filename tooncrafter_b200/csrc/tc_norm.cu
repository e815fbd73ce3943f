// tooncrafter_b200 — GroupNorm(+SiLU) and LayerNorm, channels-last fp16, fp32 statistics (HBM-bound).
//
// GroupNorm reference sites: lvdm/basics.py:76-87 (GroupNormSpecific, eps 1e-5, 4-D per frame and 5-D per clip),
// lvdm/modules/attention.py:265,331 (eps 1e-6), openaimodel3d.py:256-265 (5-D), autoencoder_dualref.py:29-32.
// LayerNorm: lvdm/modules/attention.py:225-227.
//
// Algorithmic bytes: GroupNorm = 2 reads + 1 write of the activation (statistics pass + apply pass; the second
// read hits L2 for UNet-sized tensors); LayerNorm = 1 read + 1 write.
#include <stdlib.h>

#include "tc_common.cuh"
#include "tc_host.h"

namespace {

constexpr int kGnMaxPartials = TC_GN_MAX_PARTIALS;

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 u;
    __half2 h[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    u.x = *reinterpret_cast<uint32_t*>(&h[0]);
    u.y = *reinterpret_cast<uint32_t*>(&h[1]);
    u.z = *reinterpret_cast<uint32_t*>(&h[2]);
    u.w = *reinterpret_cast<uint32_t*>(&h[3]);
    return u;
}

// ---- pass 1: per-block partial (sum, sumsq) per group -------------------------------------------------
// grid = (nblk, n_stat); block = V * rows_per_iter threads (V = C/8) rounded up to whole warps: thread t < V *
// rows_per_iter owns channel vector t % V of pixel row t / V, the threads past them only take part in the reduction.
__global__ void gn_stats_kernel(const __half* __restrict__ x, long long ldx, long long pixels_per_stat, int C, int G,
                                int rows_per_iter, float* __restrict__ partials) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    extern __shared__ float sm[];  // [rows_per_iter][2*C]: per-thread partials, reduced in a fixed order (deterministic)
    const int V = C >> 3;
    const int v = threadIdx.x % V;
    const int prow = threadIdx.x / V;
    const int s = blockIdx.y;

    float sum[8], sq[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sum[i] = sq[i] = 0.f;
    const __half* base = x + (long long)s * pixels_per_stat * ldx + (long long)v * 8;
    const long long stride = (long long)gridDim.x * rows_per_iter;
    // 4 independent 16-byte loads in flight per thread (the pass is pure HBM/L2 streaming)
    const long long pix_end = prow < rows_per_iter ? pixels_per_stat : 0;
    for (long long pix = (long long)blockIdx.x * rows_per_iter + prow; pix < pix_end; pix += 4 * stride) {
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const long long pp = pix + k * stride;
            if (pp < pixels_per_stat) u[k] = *reinterpret_cast<const uint4*>(base + pp * ldx);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (pix + k * stride < pixels_per_stat) {
                float f[8];
                unpack8(u[k], f);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    sum[i] += f[i];
                    sq[i] += f[i] * f[i];
                }
            }
        }
    }
    if (prow < rows_per_iter) {
        float* mine = sm + (long long)prow * 2 * C;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            mine[v * 8 + i] = sum[i];
            mine[C + v * 8 + i] = sq[i];
        }
    }
    __syncthreads();
    // block reduction in a fixed order (deterministic), one warp per (group, sum | sumsq) task rather than 32 threads
    // walking rows_per_iter x cpg values serially (blockDim.x is a multiple of 32: every warp is whole)
    const int cpg = C / G;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int n = rows_per_iter * cpg;
    for (int task = warp; task < 2 * G; task += nwarps) {
        const int g = task >> 1, which = task & 1;
        const float* src = sm + which * C + g * cpg;
        float a = 0.f;
        for (int e = lane; e < n; e += 32) a += src[(long long)(e / cpg) * 2 * C + (e % cpg)];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) partials[(((long long)s * gridDim.x + blockIdx.x) * G + g) * 2 + which] = a;
    }
}

// ---- pass 2: finalize statistics for this block's stat group, then normalise (+SiLU) -------------------
// grid = (blocks_per_stat, n_stat); block as gn_stats_kernel (whole warps, V * rows_per_iter of them normalise)
__global__ void gn_apply_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy,
                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                long long pixels_per_stat, int C, int G, int rows_per_iter, float eps, int silu,
                                const float* __restrict__ partials, int nblk) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    extern __shared__ float sm[];  // mean[G], rstd[G]
    float* s_mean = sm;
    float* s_rstd = sm + G;
    const int s = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int cpg = C / G;
    // 8 lanes per group: all groups of a 32-group layer are finished in one round by 8+ warps
    for (int gb = warp * 4; gb < G; gb += nwarps * 4) {     // warp-uniform trip count: the shuffles use the full mask
        const int g = gb + (lane >> 3);
        double a = 0.0, b = 0.0;
        for (int k = lane & 7; k < nblk && g < G; k += 8) {
            const float* src = partials + (((long long)s * nblk + k) * G + g) * 2;
            a += (double)src[0];
            b += (double)src[1];
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if ((lane & 7) == 0 && g < G) {
            const double cnt = (double)pixels_per_stat * (double)cpg;
            const double mean = a / cnt;
            double var = b / cnt - mean * mean;
            if (var < 0.0) var = 0.0;
            s_mean[g] = (float)mean;
            s_rstd[g] = (float)(1.0 / sqrt(var + (double)eps));
        }
    }
    __syncthreads();

    const int V = C >> 3;
    const int v = threadIdx.x % V;
    const int prow = threadIdx.x / V;
    if (prow >= rows_per_iter) return;
    float sc[8], sh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = v * 8 + i;
        const int g = c / cpg;
        const float a = s_rstd[g] * gamma[c];
        sc[i] = a;
        sh[i] = beta[c] - s_mean[g] * a;
    }
    const __half* xb = x + (long long)s * pixels_per_stat * ldx + (long long)v * 8;
    __half* yb = y + (long long)s * pixels_per_stat * ldy + (long long)v * 8;
    const long long stride = (long long)gridDim.x * rows_per_iter;
    for (long long pix = (long long)blockIdx.x * rows_per_iter + prow; pix < pixels_per_stat; pix += 4 * stride) {
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const long long pp = pix + k * stride;
            if (pp < pixels_per_stat) u[k] = *reinterpret_cast<const uint4*>(xb + pp * ldx);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const long long pp = pix + k * stride;
            if (pp < pixels_per_stat) {
                float f[8];
                unpack8(u[k], f);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float t = f[i] * sc[i] + sh[i];
                    if (silu) t = tc::silu_f(t);
                    f[i] = t;
                }
                *reinterpret_cast<uint4*>(yb + pp * ldy) = pack8(f);
            }
        }
    }
}

// ---- single-pass GroupNorm for small / medium tensors: one CTA (or a cluster of 2-8 CTAs) per (stat group, norm group) -----
// The two-kernel path pays two launches and two reads of the tensor, which dominate for the few-MB activations of UNet
// levels 2 and 3 (77 of the 166 GroupNorms of a forward).  Here the unit's elements — `cpg` contiguous
// channels of every pixel of the stat group — are loaded ONCE into registers (kVec-byte vectors, at most kMaxV per thread),
// reduced (warp shuffles -> shared memory -> fixed-order sum; across a cluster through distributed shared memory, summed in
// rank order: deterministic), normalised (+SiLU) in registers and stored.  One read, one write, one launch.
__device__ __forceinline__ float ld_dsmem_f32(const float* local_ptr, uint32_t rank) {
    float v;
    asm volatile(
        "{\n\t"
        ".reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %1, %2;\n\t"
        "ld.shared::cluster.f32 %0, [ra];\n\t"
        "}\n"
        : "=f"(v)
        : "r"(tc::smem_u32(local_ptr)), "r"(rank)
        : "memory");
    return v;
}

template <int kMaxV>
__global__ void __launch_bounds__(640, 1) gn_fused_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           long long pixels_per_stat, int C, int G, float eps, int silu, int csize) {
    tc::pdl_wait();   // no early launch_dependents (see gn_stats_kernel)
    __shared__ float s_part[2][32];      // per-warp partial {sum, sumsq}
    __shared__ float s_cta[2];           // this CTA's {sum, sumsq}: read by the cluster peers
    __shared__ float s_stat[2];          // {mean, rstd}
    const int cpg = C / G;
    const int vpp = cpg >> 3;                         // 16-byte vectors per pixel of this norm group
    const int unit = (int)blockIdx.x / csize;         // (stat group, norm group)
    const uint32_t rank = csize > 1 ? tc::cluster_ctarank() : 0u;
    const int s = unit / G, g = unit - s * G;
    const int T = (int)blockDim.x;                    // a multiple of vpp: thread t always owns channel vector t % vpp
    const int k = (int)threadIdx.x % vpp;
    const long long total_v = pixels_per_stat * vpp;
    const long long per_cta = (total_v + csize - 1) / csize;
    long long v_begin = (long long)rank * per_cta;
    v_begin -= v_begin % vpp;                         // whole pixels per CTA (keeps t % vpp == channel vector)
    long long v_end = (long long)(rank + 1) * per_cta;
    v_end -= v_end % vpp;
    if ((int)rank == csize - 1) v_end = total_v;
    const __half* xb = x + (long long)s * pixels_per_stat * ldx + (long long)g * cpg + (long long)k * 8;
    __half* yb = y + (long long)s * pixels_per_stat * ldy + (long long)g * cpg + (long long)k * 8;

    uint4 u[kMaxV];
    float sum = 0.f, sq = 0.f;
    // sums are taken about a pivot, the unit's first element (the same for every CTA of the cluster): E[x^2] - E[x]^2
    // from fp32 sums of raw values cancels when the mean is large against the spread, sums about a value within a few
    // standard deviations of the mean do not
    const float pivot = __half2float(x[(long long)s * pixels_per_stat * ldx + (long long)g * cpg]);
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
        const long long v = v_begin + threadIdx.x + (long long)i * T;
        if (v < v_end) u[i] = *reinterpret_cast<const uint4*>(xb + (v / vpp) * ldx);
    }
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
        const long long v = v_begin + threadIdx.x + (long long)i * T;
        if (v < v_end) {
            float f[8];
            unpack8(u[i], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float d = f[j] - pivot;
                sum += d;
                sq += d * d;
            }
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = T >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    if (lane == 0) {
        s_part[0][warp] = sum;
        s_part[1][warp] = sq;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float a = 0.f, b = 0.f;
        for (int w = 0; w < nwarps; ++w) {
            a += s_part[0][w];
            b += s_part[1][w];
        }
        s_cta[0] = a;
        s_cta[1] = b;
    }
    if (csize > 1) tc::cluster_sync_all(); else __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        if (csize > 1) {
            for (int r = 0; r < csize; ++r) {                // rank order: every CTA of the cluster computes the same bits
                a += (double)ld_dsmem_f32(&s_cta[0], (uint32_t)r);
                b += (double)ld_dsmem_f32(&s_cta[1], (uint32_t)r);
            }
        } else {
            a = s_cta[0];
            b = s_cta[1];
        }
        const double cnt = (double)pixels_per_stat * (double)cpg;
        const double dmean = a / cnt;                  // mean - pivot
        double var = b / cnt - dmean * dmean;
        if (var < 0.0) var = 0.0;
        s_stat[0] = (float)((double)pivot + dmean);
        s_stat[1] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __syncthreads();
    const float mean = s_stat[0], rstd = s_stat[1];
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = g * cpg + k * 8 + j;
        const float a = rstd * gamma[c];
        sc[j] = a;
        sh[j] = beta[c] - mean * a;
    }
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
        const long long v = v_begin + threadIdx.x + (long long)i * T;
        if (v < v_end) {
            float f[8];
            unpack8(u[i], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float t = f[j] * sc[j] + sh[j];
                if (silu) t = tc::silu_f(t);
                f[j] = t;
            }
            *reinterpret_cast<uint4*>(yb + (v / vpp) * ldy) = pack8(f);
        }
    }
    if (csize > 1) tc::cluster_sync_all();     // peers may still be reading this CTA's s_cta
}

// ---- LayerNorm: one warp per row, row kept in registers ------------------------------------------------
template <int kMaxVec>
__global__ void layernorm_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, int rows, int C,
                                 float eps) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int V = C >> 3;
    const __half* xr = x + (long long)warp * ldx;
    float f[kMaxVec][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < V) {
            const uint4 u = *reinterpret_cast<const uint4*>(xr + v * 8);
            unpack8(u, f[i]);
#pragma unroll
            for (int j = 0; j < 8; ++j) sum += f[i][j];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < V) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float d = f[i][j] - mean;
                sq += d * d;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / (float)C + eps);
    __half* yr = y + (long long)warp * ldy;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < V) {
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = v * 8 + j;
                o[j] = (f[i][j] - mean) * rstd * gamma[c] + beta[c];
            }
            *reinterpret_cast<uint4*>(yr + v * 8) = pack8(o);
        }
    }
}

// ---- LayerNorm statistics only: (mean, rstd) per row; the normalisation is folded into the consuming GEMM ----
template <int kMaxVec>
__global__ void row_stats_kernel(const __half* __restrict__ x, long long ldx, int rows, int C, float eps,
                                 float2* __restrict__ stats) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int V = C >> 3;
    const __half* xr = x + (long long)warp * ldx;
    float f[kMaxVec][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < V) {
            const uint4 u = *reinterpret_cast<const uint4*>(xr + v * 8);
            unpack8(u, f[i]);
#pragma unroll
            for (int j = 0; j < 8; ++j) sum += f[i][j];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < V) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float d = f[i][j] - mean;
                sq += d * d;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if (lane == 0) stats[warp] = make_float2(mean, rsqrtf(sq / (float)C + eps));
}

}  // namespace

extern "C" int tc_row_stats(const void* x, long long ldx, int rows, int C, float eps, float* stats, void* stream_v) {
    using namespace tc_host;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && stats, "tc_row_stats: null pointer");
    TC_CHECK_ARG(C > 0 && C % 8 == 0 && C <= 2048 && ldx % 8 == 0 && rows > 0, "tc_row_stats: bad shape");
    TC_CHECK_ARG(ldx >= C, "tc_row_stats: ldx must be at least C");
    TC_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(stats) & 7) == 0,
                 "tc_row_stats: x must be 16-byte and stats 8-byte aligned");
    const int threads = 256;
    const int blocks = (rows + 7) / 8;
    const __half* xp = reinterpret_cast<const __half*>(x);
    float2* sp = reinterpret_cast<float2*>(stats);
    if (C <= 512)
        tc_host::launch(row_stats_kernel<2>, dim3(blocks), dim3(threads), 0, stream, 1, xp, ldx, rows, C, eps, sp);
    else if (C <= 1280)
        tc_host::launch(row_stats_kernel<5>, dim3(blocks), dim3(threads), 0, stream, 1, xp, ldx, rows, C, eps, sp);
    else
        tc_host::launch(row_stats_kernel<8>, dim3(blocks), dim3(threads), 0, stream, 1, xp, ldx, rows, C, eps, sp);
    count_launch();
    TC_CHECK_LAUNCH("row_stats_kernel");
    return TC_OK;
}

extern "C" int tc_groupnorm(const void* x, long long ldx, void* y, long long ldy, const float* gamma,
                            const float* beta, int frames, int frames_per_stat, int hw, int C, int G, float eps,
                            int silu, float* ws, void* stream_v) {
    using namespace tc_host;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && gamma && beta && ws, "tc_groupnorm: null pointer");
    TC_CHECK_ARG(C > 0 && C % 8 == 0 && G > 0 && C % G == 0, "tc_groupnorm: need C % 8 == 0 and C % G == 0");
    TC_CHECK_ARG(C / 8 <= 512, "tc_groupnorm: C too large (max 4096)");
    TC_CHECK_ARG(frames > 0 && frames_per_stat > 0 && frames % frames_per_stat == 0 && hw > 0,
                 "tc_groupnorm: bad frame counts");
    TC_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0, "tc_groupnorm: strides must be multiples of 8");
    TC_CHECK_ARG(ldx >= C && ldy >= C, "tc_groupnorm: ldx and ldy must be at least C");
    TC_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0,
                 "tc_groupnorm: x and y must be 16-byte aligned");
    const int n_stat = frames / frames_per_stat;
    const long long pps = (long long)frames_per_stat * hw;
    {
        // single-pass path: (C / G) % 8 == 0 (16-byte vectors per norm group) and the unit fits the registers of <= 8 CTAs
        static const char* fused_env = getenv("TC_GN_FUSED");     // "0" disables (A/B testing)
        const int cpg = C / G;
        constexpr int kMaxV = 8;
        // (large tensors stay on the streaming two-kernel path: 5+ TB/s there, and a unit's 16-80 bytes per pixel row
        // would be a poor access pattern at hundreds of megabytes)
        if (cpg % 8 == 0 && (long long)frames * hw * C * 2 <= (16LL << 20) && !(fused_env && fused_env[0] == '0')) {
            const int vpp = cpg / 8;
            const long long total_v = pps * vpp;
            int threads = (640 / (32 * vpp)) * (32 * vpp);            // multiple of 32 and of vpp, <= 640
            if (32 % vpp == 0) threads = 640;
            if (threads >= 32 && total_v <= 8LL * threads * kMaxV) {
                int csize = 1;
                while ((long long)csize * threads * kMaxV < total_v + (long long)csize * (vpp + 1)) ++csize;   // whole pixels per CTA
                // (a large tensor would need several waves of one-per-SM CTAs: it stays on the two-kernel path)
                const long long n_units = (long long)n_stat * G;
                if (csize <= 8 && (csize == 1 || n_units * csize <= 2LL * sm_count())) {
                    // small units: shrink the block to what the unit needs (several units resident per SM); with many units
                    // (per-frame statistics: 1024 of them) fewer, fuller threads keep the grid near one wave
                    if (csize == 1) {
                        const int step = (32 % vpp == 0) ? 32 : 32 * vpp;
                        const int per_thread = n_units >= 4LL * sm_count() ? kMaxV : kMaxV / 2;
                        const long long need = (total_v + per_thread - 1) / per_thread;
                        int t2 = (int)((need + step - 1) / step) * step;
                        if (t2 < step) t2 = step;
                        if (t2 < threads) threads = t2;
                    }
                    tc_host::launch(gn_fused_kernel<kMaxV>, dim3((unsigned)(n_stat * G * csize)), dim3(threads), 0, stream, csize,
                                    reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<__half*>(y), ldy, gamma, beta, pps, C, G,
                                    eps, silu, csize);
                    count_launch();
                    TC_CHECK_LAUNCH("gn_fused_kernel");
                    return TC_OK;
                }
            }
        }
    }
    const int V = C / 8;
    int k = 512 / V;
    if (k < 1) k = 1;
    // k pixel rows of V vectors per block, rounded up to whole warps (the warp-per-task reductions shuffle over all 32
    // lanes); the surplus threads load nothing
    const int threads = (V * k + 31) / 32 * 32;
    // small tensors are latency-bound (a chain of dependent load rounds per thread): spread them over as many blocks as
    // one round of 4 loads per thread allows; large ones are capped to one resident wave below
    long long want = (pps + (long long)k * 4 - 1) / ((long long)k * 4);
    int nblk = (int)(want < 1 ? 1 : want);
    // exactly one resident wave (2 blocks of <= 512 threads per SM): one block more than that runs as two waves
    int cap = (2 * sm_count()) / n_stat;
    if (cap < 1) cap = 1;
    if (cap > kGnMaxPartials) cap = kGnMaxPartials;
    if (nblk > cap) nblk = cap;
    tc_host::launch(gn_stats_kernel, dim3(dim3(nblk, n_stat)), dim3(threads), (size_t)k * 2 * C * sizeof(float), stream, 1, 
        reinterpret_cast<const __half*>(x), ldx, pps, C, G, k, ws);
    count_launch();
    TC_CHECK_LAUNCH("gn_stats_kernel");
    long long want2 = (pps + (long long)k * 4 - 1) / ((long long)k * 4);
    int nblk2 = (int)(want2 < 1 ? 1 : want2);
    // one wave as well: every block pays the fp64 finalize prologue once
    int cap2 = (2 * sm_count()) / n_stat;
    if (cap2 < 1) cap2 = 1;
    if (nblk2 > cap2) nblk2 = cap2;
    tc_host::launch(gn_apply_kernel, dim3(dim3(nblk2, n_stat)), dim3(threads), 2 * G * sizeof(float), stream, 1, 
        reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<__half*>(y), ldy, gamma, beta, pps, C, G, k, eps, silu,
        ws, nblk);
    count_launch();
    TC_CHECK_LAUNCH("gn_apply_kernel");
    return TC_OK;
}

extern "C" int tc_layernorm(const void* x, long long ldx, void* y, long long ldy, const float* gamma,
                            const float* beta, int rows, int C, float eps, void* stream_v) {
    using namespace tc_host;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && gamma && beta, "tc_layernorm: null pointer");
    TC_CHECK_ARG(C > 0 && C % 8 == 0 && C <= 2048, "tc_layernorm: need C % 8 == 0 and C <= 2048");
    TC_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0 && rows > 0, "tc_layernorm: bad strides/rows");
    TC_CHECK_ARG(ldx >= C && ldy >= C, "tc_layernorm: ldx and ldy must be at least C");
    TC_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0,
                 "tc_layernorm: x and y must be 16-byte aligned");
    const int threads = 256;
    const int blocks = (rows + 7) / 8;
    const __half* xp = reinterpret_cast<const __half*>(x);
    __half* yp = reinterpret_cast<__half*>(y);
    if (C <= 512)
        tc_host::launch(layernorm_kernel<2>, dim3(blocks), dim3(threads), 0, stream, 1, xp, ldx, yp, ldy, gamma, beta, rows, C, eps);
    else if (C <= 1280)
        tc_host::launch(layernorm_kernel<5>, dim3(blocks), dim3(threads), 0, stream, 1, xp, ldx, yp, ldy, gamma, beta, rows, C, eps);
    else
        tc_host::launch(layernorm_kernel<8>, dim3(blocks), dim3(threads), 0, stream, 1, xp, ldx, yp, ldy, gamma, beta, rows, C, eps);
    count_launch();
    TC_CHECK_LAUNCH("layernorm_kernel");
    return TC_OK;
}
