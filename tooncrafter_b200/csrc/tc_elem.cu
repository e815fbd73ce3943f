// tooncrafter_b200 — data-movement / elementwise kernels, tiny linears and the fused DDIM update (HBM-bound).
// Reference sites are listed per entry point in include/tooncrafter_b200.h.
#include <stdlib.h>

#include "tc_common.cuh"
#include "tc_host.h"

namespace {

__device__ __forceinline__ uint4 ld16(const void* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void st16(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }

// ------------------------------------------------------------------------------------------------ layout
__global__ void ncthw_to_cl_kernel(const float* __restrict__ x, __half* __restrict__ y, int B, int C, int T, int H,
                                   int W, int Cpad, int coff, float scale) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const long long npix = (long long)B * T * H * W;
    const long long thw = (long long)T * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < npix;
         i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / thw, r = i - b * thw;
        const float* src = x + b * C * thw + r;
        __half* dst = y + i * Cpad + coff;
        for (int c = 0; c < C; ++c) dst[c] = __float2half_rn(src[(long long)c * thw] * scale);
    }
}

// Tiled form for wide tensors (C % 64 == 0: the decoder's reference-frame feature maps, 128-512 channels): a 32-pixel x
// 64-channel tile goes through shared memory, so the fp32 planes are read 128 bytes at a time AND the channels-last rows are
// written as 16-byte vectors (the per-pixel loop above writes 2 bytes per thread per instruction).  grid = (pixel tiles,
// channel tiles, B), 256 threads.
__global__ void ncthw_to_cl_tiled_kernel(const float* __restrict__ x, __half* __restrict__ y, int C, long long thw, int Cpad,
                                         int coff, float scale) {
    tc::pdl_wait();
    __shared__ float tile[64][33];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long r0 = (long long)blockIdx.x * 32;
    const int c0 = (int)blockIdx.y * 64;
    const long long b = blockIdx.z;
    const float* src = x + (b * C + c0) * thw + r0 + lane;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = warp + 8 * k;
        tile[c][lane] = (r0 + lane < thw) ? src[(long long)c * thw] * scale : 0.f;
    }
    __syncthreads();
    const int p = threadIdx.x >> 3, chunk = threadIdx.x & 7;          // 32 pixels x 8 chunks of 8 channels
    if (r0 + p < thw) {
        __half2 h[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(tile[chunk * 8 + 2 * j][p], tile[chunk * 8 + 2 * j + 1][p]);
        uint4 u;
        u.x = *reinterpret_cast<uint32_t*>(&h[0]);
        u.y = *reinterpret_cast<uint32_t*>(&h[1]);
        u.z = *reinterpret_cast<uint32_t*>(&h[2]);
        u.w = *reinterpret_cast<uint32_t*>(&h[3]);
        *reinterpret_cast<uint4*>(y + (b * thw + r0 + p) * Cpad + coff + c0 + chunk * 8) = u;
    }
}

template <typename OutT>
__global__ void cl_to_ncthw_kernel(const __half* __restrict__ x, long long ldx, OutT* __restrict__ y, int B, int C,
                                   int T, int H, int W) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const long long npix = (long long)B * T * H * W;
    const long long thw = (long long)T * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < npix;
         i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / thw, r = i - b * thw;
        const __half* src = x + i * ldx;
        OutT* dst = y + b * C * thw + r;
        for (int c = 0; c < C; ++c) {
            if constexpr (sizeof(OutT) == 2)
                dst[(long long)c * thw] = src[c];
            else
                dst[(long long)c * thw] = __half2float(src[c]);
        }
    }
}

__global__ void upsample2x_kernel(const __half* __restrict__ x, __half* __restrict__ y, int N, int H, int W, int C) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int V = C >> 3;
    const long long total = (long long)N * (2 * H) * (2 * W) * V;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(i % V);
        long long p = i / V;
        const int ox = (int)(p % (2 * W));
        p /= (2 * W);
        const int oy = (int)(p % (2 * H));
        const long long n = p / (2 * H);
        const __half* src = x + (((n * H + (oy >> 1)) * W + (ox >> 1)) * (long long)C) + v * 8;
        st16(y + i * 8, ld16(src));
    }
}

// y[ph][n][h2][w2][c] = x[n][2*h2 + (ph>>1)][2*w2 + (ph&1)][c]
__global__ void phase_split2_kernel(const __half* __restrict__ x, __half* __restrict__ y, int N, int H, int W,
                                    int C) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int V = C >> 3;
    const int H2 = H >> 1, W2 = W >> 1;
    const long long total = (long long)4 * N * H2 * W2 * V;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(i % V);
        long long p = i / V;
        const int w2 = (int)(p % W2);
        p /= W2;
        const int h2 = (int)(p % H2);
        p /= H2;
        const long long n = p % N;
        const int ph = (int)(p / N);
        const __half* src = x + (((n * H + (2 * h2 + (ph >> 1))) * W + (2 * w2 + (ph & 1))) * (long long)C) + v * 8;
        st16(y + i * 8, ld16(src));
    }
}

__global__ void copy2d_kernel(const __half* __restrict__ src, long long lds, __half* __restrict__ dst, long long ldd,
                              long long rows, int cols) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int V = cols >> 3;
    const long long total = rows * V;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / V;
        const int v = (int)(i - r * V);
        st16(dst + r * ldd + v * 8, ld16(src + r * lds + v * 8));
    }
}

// y = GELU(x) (exact erf form, nn.GELU default) on a strided 2-D half matrix, in place allowed
__global__ void gelu2d_kernel(const __half* __restrict__ x, long long ldx, __half* y, long long ldy, long long rows, int cols) {
    tc::pdl_wait();
    const int V = cols >> 3;
    const long long total = rows * V;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / V;
        const int v = (int)(i - r * V);
        uint4 a = ld16(x + r * ldx + v * 8);
        __half2* ha = reinterpret_cast<__half2*>(&a);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = __half22float2(ha[k]);
            ha[k] = __floats2half2_rn(tc::gelu_erf_f(f.x), tc::gelu_erf_f(f.y));
        }
        st16(y + r * ldy + v * 8, a);
    }
}

__global__ void add2d_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy,
                             long long rows, int cols) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int V = cols >> 3;
    const long long total = rows * V;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / V;
        const int v = (int)(i - r * V);
        uint4 a = ld16(x + r * ldx + v * 8);
        uint4 b = ld16(y + r * ldy + v * 8);
        __half2* ha = reinterpret_cast<__half2*>(&a);
        __half2* hb = reinterpret_cast<__half2*>(&b);
#pragma unroll
        for (int k = 0; k < 4; ++k) hb[k] = __hadd2(hb[k], ha[k]);
        st16(y + r * ldy + v * 8, b);
    }
}

// ------------------------------------------------------------------------------------------------ tiny linears
// sinusoidal embedding: out[b][0:half] = cos(t*f_i), out[b][half:2*half] = sin(t*f_i), f_i = exp(-ln(1e4)*i/half)
__global__ void sincos_kernel(const float* __restrict__ t, int B, int dim, float* __restrict__ out) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int half = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, k = i - b * half;
    const float freq = expf(-9.210340371976184f * (float)k / (float)half);
    const float a = t[b] * freq;
    out[(long long)b * dim + k] = cosf(a);
    out[(long long)b * dim + half + k] = sinf(a);
    if ((dim & 1) && k == 0) out[(long long)b * dim + dim - 1] = 0.f;
}

// y[b][j] (+)= sum_k act(x[b][k]) * W[j][k] + bias[j]   one warp per output column j, all B rows (B <= 8 per pass)
template <typename OutT>
__global__ void small_linear_kernel(const float* __restrict__ x, int B, int K, const __half* __restrict__ w,
                                    const float* __restrict__ bias, int J, OutT* __restrict__ y, long long ldy,
                                    int silu_in, int accumulate) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (j >= J) return;
    const __half* wr = w + (long long)j * K;
    for (int b0 = 0; b0 < B; b0 += 8) {
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        for (int k = lane * 8; k < K; k += 32 * 8) {
            const uint4 u = ld16(wr + k);
            const __half2* h = reinterpret_cast<const __half2*>(&u);
            float wf[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = __half22float2(h[i]);
                wf[2 * i] = f.x;
                wf[2 * i + 1] = f.y;
            }
#pragma unroll
            for (int bi = 0; bi < 8; ++bi) {
                if (b0 + bi < B) {
                    const float* xr = x + (long long)(b0 + bi) * K + k;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        float xv = xr[i];
                        if (silu_in) xv = xv / (1.0f + expf(-xv));
                        acc[bi] += xv * wf[i];
                    }
                }
            }
        }
#pragma unroll
        for (int bi = 0; bi < 8; ++bi) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[bi] += __shfl_xor_sync(0xffffffffu, acc[bi], o);
        }
        if (lane == 0) {
            for (int bi = 0; bi < 8 && b0 + bi < B; ++bi) {
                float v = acc[bi] + (bias ? bias[j] : 0.f);
                OutT* dst = y + (long long)(b0 + bi) * ldy + j;
                if constexpr (sizeof(OutT) == 2) {
                    *dst = __float2half_rn(v);
                } else {
                    if (accumulate) v += *dst;
                    *dst = v;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ DDIM step
// classifier-free-guidance combine in fp16 arithmetic (each torch op rounds to half: ddim.py:226)
__device__ __forceinline__ __half cfg_combine(__half ec, __half euc, float s) {
    const __half d = __float2half_rn(__half2float(ec) - __half2float(euc));
    const __half m = __float2half_rn(s * __half2float(d));
    return __float2half_rn(__half2float(euc) + __half2float(m));
}

// three-way guidance of the multi-condition sampler (ddim_multiplecond.py:229):
//   e_uc + cfg_img * (e_img - e_uc) + s * (e_c - e_img), every torch op rounding to half, left to right
__device__ __forceinline__ __half cfg_combine3(__half ec, __half euc, __half eimg, float s, float cfg_img) {
    const __half d1 = __float2half_rn(__half2float(eimg) - __half2float(euc));
    const __half m1 = __float2half_rn(cfg_img * __half2float(d1));
    const __half a1 = __float2half_rn(__half2float(euc) + __half2float(m1));
    const __half d2 = __float2half_rn(__half2float(ec) - __half2float(eimg));
    const __half m2 = __float2half_rn(s * __half2float(d2));
    return __float2half_rn(__half2float(a1) + __half2float(m2));
}
// e_img == nullptr: the two-way combine of ddim.py:226; coef[8] (cfg_img) is only read for the three-way form
__device__ __forceinline__ __half cfg_any(const __half* ec, const __half* eu, const __half* ei, long long i, float s,
                                          float cfg_img) {
    return ei ? cfg_combine3(ec[i], eu[i], ei[i], s, cfg_img) : cfg_combine(ec[i], eu[i], s);
}

// partial sums for std(e_c) and std(v): ws[b][blk][4] = {sum_ec, sumsq_ec, sum_v, sumsq_v} (double)
__global__ void ddim_reduce_kernel(const __half* __restrict__ e_c, const __half* __restrict__ e_uc,
                                   const __half* __restrict__ e_img, const float* __restrict__ coef, long long n,
                                   double* __restrict__ ws) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int b = blockIdx.y;
    const float s = coef[0];
    const float cfg_img = e_img ? coef[8] : 0.f;
    const __half* ec = e_c + (long long)b * n;
    const __half* eu = e_uc + (long long)b * n;
    const __half* ei = e_img ? e_img + (long long)b * n : nullptr;
    double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float c = __half2float(ec[i]);
        const float v = __half2float(cfg_any(ec, eu, ei, i, s, cfg_img));
        a0 += c;
        a1 += (double)c * c;
        a2 += v;
        a3 += (double)v * v;
    }
    __shared__ double red[4][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o);
        a3 += __shfl_xor_sync(0xffffffffu, a3, o);
    }
    if (lane == 0) {
        red[0][warp] = a0;
        red[1][warp] = a1;
        red[2][warp] = a2;
        red[3][warp] = a3;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        double t = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[threadIdx.x][w];
        ws[((long long)b * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = t;
    }
}

// kDpm (DPM-Solver++(2M), prev_pred_x0 = the previous step's pred_x0): x_prev += c * (pred_x0 - prev_pred_x0), with
// c = coef[8] (coef[9] with e_img) and each op rounded on its own as torch's fp32 arithmetic.  c == 0 marks a first-order
// step: the term is skipped and prev_pred_x0 is not read.  Without kDpm this is the DDIM update, and prev_pred_x0 unused.
template <bool kDpm>
__global__ void ddim_update_kernel(const __half* __restrict__ e_c, const __half* __restrict__ e_uc,
                                   const __half* __restrict__ e_img, const float* __restrict__ x, const float* __restrict__ noise,
                                   float* __restrict__ x_prev, float* __restrict__ pred_x0,
                                   const float* __restrict__ coef, long long n, const double* __restrict__ ws,
                                   int nblk, const float* __restrict__ prev_pred_x0) {
    tc::pdl_wait();   // no early launch_dependents: waiting successor CTAs would squat on this kernel's SM slots
    const int b = blockIdx.y;
    const float s = coef[0], phi = coef[1], sqrt_ac = coef[2], sqrt_1mac = coef[3], rescale = coef[4],
                sqrt_aprev = coef[5], dir_coef = coef[6], sigma = coef[7];
    __shared__ float s_ratio;
    if (threadIdx.x == 0) {
        float ratio = 1.0f;
        if (phi > 0.f) {
            double t[4] = {0, 0, 0, 0};
            for (int k = 0; k < nblk; ++k)
                for (int j = 0; j < 4; ++j) t[j] += ws[((long long)b * nblk + k) * 4 + j];
            const double dn = (double)n;
            const double var_c = (t[1] - t[0] * t[0] / dn) / (dn - 1.0);
            const double var_v = (t[3] - t[2] * t[2] / dn) / (dn - 1.0);
            // torch.std on fp16 tensors returns fp16; the ratio is an fp16 division (utils_diffusion.py:152-155)
            const __half std_c = __float2half_rn((float)sqrt(var_c > 0 ? var_c : 0));
            const __half std_v = __float2half_rn((float)sqrt(var_v > 0 ? var_v : 0));
            ratio = __half2float(__float2half_rn(__half2float(std_c) / __half2float(std_v)));
        }
        s_ratio = ratio;
    }
    __syncthreads();
    const float ratio = s_ratio;
    const long long off = (long long)b * n;
    const float cfg_img = e_img ? coef[8] : 0.f;
    const float c2 = kDpm ? coef[e_img ? 9 : 8] : 0.f;
    const __half* ei = e_img ? e_img + off : nullptr;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        __half vh = cfg_any(e_c + off, e_uc + off, ei, i, s, cfg_img);
        if (phi > 0.f) {
            const __half resc = __float2half_rn(__half2float(vh) * ratio);
            const __half t1 = __float2half_rn(phi * __half2float(resc));
            const __half t2 = __float2half_rn((1.0f - phi) * __half2float(vh));
            vh = __float2half_rn(__half2float(t1) + __half2float(t2));
        }
        const float v = __half2float(vh);
        const float xv = x[off + i];
        const float eps = sqrt_ac * v + sqrt_1mac * xv;
        float x0 = sqrt_ac * xv - sqrt_1mac * v;
        x0 *= rescale;
        pred_x0[off + i] = x0;
        float xp = sqrt_aprev * x0 + dir_coef * eps + sigma * noise[off + i];
        if (kDpm && c2 != 0.f) xp = __fadd_rn(xp, __fmul_rn(c2, __fsub_rn(x0, prev_pred_x0[off + i])));
        x_prev[off + i] = xp;
    }
}

// ------------------------------------------------------------------------------------------------ video output
// One channel value of the reference's save path (inference.py:148-153), in torch's fp32 op order with no contraction:
// clamp(x, -1, 1) -> (v + 1) / 2 -> v * 255 -> uint8 (truncation toward zero; v is in [0, 255]).
__device__ __forceinline__ uint32_t to_u8(__half h) {
    float v = fminf(fmaxf(__half2float(h), -1.0f), 1.0f);
    v = __fdiv_rn(__fadd_rn(v, 1.0f), 2.0f);
    v = __fmul_rn(v, 255.0f);
    return __float2uint_rz(v);
}

// Output frame f (of [f_begin, f_end)) of one segment, written as out[f - f_begin][p][c] (NTHWC uint8).  Source: the
// 16-frame decode x16 [T][3][HW], except frames T/2-1 and T/2, which come from frames T/2-2 and T/2-1 of the 14-frame
// decode x14 [T-2][3][HW] when it is given (inference.py:270).  One thread per group of 8 pixels of one frame: with
// vec, three 16-byte channel-plane loads and three 8-byte stores of the 24 packed bytes; otherwise a scalar loop.
__global__ void video_u8_kernel(const __half* __restrict__ x16, const __half* __restrict__ x14, int T, long long HW,
                                int f_begin, int n_frames, uint8_t* __restrict__ out, int vec) {
    tc::pdl_wait();
    const long long groups = (HW + 7) / 8;
    const long long total = groups * n_frames;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int fo = (int)(i / groups);
        const long long p0 = (i - (long long)fo * groups) * 8;
        const int f = f_begin + fo;
        const bool mid = x14 != nullptr && (f == T / 2 - 1 || f == T / 2);
        const __half* src = mid ? x14 + (long long)(f - 1) * 3 * HW : x16 + (long long)f * 3 * HW;
        uint8_t* dst = out + ((long long)fo * HW + p0) * 3;
        if (vec) {
            uint4 c[3];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) c[ch] = ld16(src + ch * HW + p0);
            const __half* h0 = reinterpret_cast<const __half*>(&c[0]);
            const __half* h1 = reinterpret_cast<const __half*>(&c[1]);
            const __half* h2 = reinterpret_cast<const __half*>(&c[2]);
            uint32_t w[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t u[3] = {to_u8(h0[k]), to_u8(h1[k]), to_u8(h2[k])};
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const int b = 3 * k + ch;                  // byte b of the 24 packed bytes
                    w[b >> 2] |= u[ch] << (8 * (b & 3));
                }
            }
            uint2* d2 = reinterpret_cast<uint2*>(dst);
            d2[0] = make_uint2(w[0], w[1]);
            d2[1] = make_uint2(w[2], w[3]);
            d2[2] = make_uint2(w[4], w[5]);
        } else {
            const int np = (int)min(8LL, HW - p0);
            for (int k = 0; k < np; ++k)
                for (int ch = 0; ch < 3; ++ch) dst[3 * k + ch] = (uint8_t)to_u8(src[ch * HW + p0 + k]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ forward diffusion
// Row b = blockIdx.y of x [B][n], in place, with a = coef[2b], c = coef[2b+1]:
//   q = clean ? x0 : a*x0 + c*noise                  (q_sample / stochastic_encode, ddpm3d.py:306-309, ddim.py:309-318)
//   x = mask ? q*m + (1 - m)*x : q                   (the masked step blend of ddim.py:172-180)
// Every multiply and add rounded on its own, in torch's op order, so the result is torch's fp32 arithmetic bit for bit.
__global__ void q_sample_kernel(float* x, const float* __restrict__ x0, const float* __restrict__ noise,
                                const float* __restrict__ mask, const float* __restrict__ coef, int clean,
                                long long n) {
    tc::pdl_wait();
    const int b = blockIdx.y;
    const float a = clean ? 0.f : coef[2 * b], c = clean ? 0.f : coef[2 * b + 1];
    const long long off = (long long)b * n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float q = clean ? x0[off + i] : __fadd_rn(__fmul_rn(a, x0[off + i]), __fmul_rn(c, noise[off + i]));
        float r = q;
        if (mask) {
            const float m = mask[off + i];
            r = __fadd_rn(__fmul_rn(q, m), __fmul_rn(__fsub_rn(1.0f, m), x[off + i]));
        }
        x[off + i] = r;
    }
}

inline int grid_for(long long total, int threads, int max_blocks) {
    long long g = (total + threads - 1) / threads;
    if (g > max_blocks) g = max_blocks;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace

using namespace tc_host;

extern "C" int tc_ncthw_to_cl(const float* x, void* y, int B, int C, int T, int H, int W, int Cpad, int coff,
                              float scale, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && B > 0 && C > 0 && T > 0 && H > 0 && W > 0, "tc_ncthw_to_cl: bad arguments");
    TC_CHECK_ARG(coff >= 0 && coff + C <= Cpad, "tc_ncthw_to_cl: channel slice out of range");
    const long long npix = (long long)B * T * H * W;
    const long long thw = (long long)T * H * W;
    static const char* tiled_env = getenv("TC_NCTHW_TILED");   // "0" keeps the per-pixel kernel (A/B testing)
    if (C % 64 == 0 && Cpad % 8 == 0 && coff % 8 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 && B <= 65535 &&
        !(tiled_env && tiled_env[0] == '0')) {
        tc_host::launch(ncthw_to_cl_tiled_kernel, dim3((unsigned)((thw + 31) / 32), (unsigned)(C / 64), (unsigned)B), dim3(256), 0, stream, 1, x,
                        reinterpret_cast<__half*>(y), C, thw, Cpad, coff, scale);
        count_launch();
        TC_CHECK_LAUNCH("ncthw_to_cl_tiled_kernel");
        return TC_OK;
    }
    tc_host::launch(ncthw_to_cl_kernel, dim3(grid_for(npix, 256, 8 * sm_count())), dim3(256), 0, stream, 1, x, reinterpret_cast<__half*>(y), B,
                                                                                C, T, H, W, Cpad, coff, scale);
    count_launch();
    TC_CHECK_LAUNCH("ncthw_to_cl_kernel");
    return TC_OK;
}

extern "C" int tc_cl_to_ncthw(const void* x, long long ldx, void* y, int out_fp32, int B, int C, int T, int H, int W,
                              void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && B > 0 && C > 0 && T > 0 && H > 0 && W > 0 && ldx >= C, "tc_cl_to_ncthw: bad arguments");
    const long long npix = (long long)B * T * H * W;
    const int g = grid_for(npix, 256, 8 * sm_count());
    if (out_fp32)
        tc_host::launch(cl_to_ncthw_kernel<float>, dim3(g), dim3(256), 0, stream, 1, reinterpret_cast<const __half*>(x), ldx,
                                                         reinterpret_cast<float*>(y), B, C, T, H, W);
    else
        tc_host::launch(cl_to_ncthw_kernel<__half>, dim3(g), dim3(256), 0, stream, 1, reinterpret_cast<const __half*>(x), ldx,
                                                          reinterpret_cast<__half*>(y), B, C, T, H, W);
    count_launch();
    TC_CHECK_LAUNCH("cl_to_ncthw_kernel");
    return TC_OK;
}

extern "C" int tc_upsample2x(const void* x, void* y, int N, int H, int W, int C, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "tc_upsample2x: bad arguments");
    const long long total = (long long)N * 4 * H * W * (C / 8);
    tc_host::launch(upsample2x_kernel, dim3(grid_for(total, 256, 16 * sm_count())), dim3(256), 0, stream, 1, 
        reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), N, H, W, C);
    count_launch();
    TC_CHECK_LAUNCH("upsample2x_kernel");
    return TC_OK;
}

extern "C" int tc_phase_split2(const void* x, void* y, int N, int H, int W, int C, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && H % 2 == 0 && W % 2 == 0,
                 "tc_phase_split2: bad arguments (H, W must be even, C % 8 == 0)");
    const long long total = (long long)N * H * W * (C / 8);
    tc_host::launch(phase_split2_kernel, dim3(grid_for(total, 256, 16 * sm_count())), dim3(256), 0, stream, 1, 
        reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), N, H, W, C);
    count_launch();
    TC_CHECK_LAUNCH("phase_split2_kernel");
    return TC_OK;
}

extern "C" int tc_copy2d(const void* src, long long lds, void* dst, long long ldd, long long rows, int cols,
                         void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(src && dst && rows > 0 && cols > 0 && cols % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0,
                 "tc_copy2d: bad arguments");
    tc_host::launch(copy2d_kernel, dim3(grid_for(rows * (cols / 8), 256, 16 * sm_count())), dim3(256), 0, stream, 1, 
        reinterpret_cast<const __half*>(src), lds, reinterpret_cast<__half*>(dst), ldd, rows, cols);
    count_launch();
    TC_CHECK_LAUNCH("copy2d_kernel");
    return TC_OK;
}

extern "C" int tc_add2d(const void* x, long long ldx, void* y, long long ldy, long long rows, int cols,
                        void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0,
                 "tc_add2d: bad arguments");
    tc_host::launch(add2d_kernel, dim3(grid_for(rows * (cols / 8), 256, 16 * sm_count())), dim3(256), 0, stream, 1, 
        reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<__half*>(y), ldy, rows, cols);
    count_launch();
    TC_CHECK_LAUNCH("add2d_kernel");
    return TC_OK;
}

extern "C" int tc_gelu2d(const void* x, long long ldx, void* y, long long ldy, long long rows, int cols,
                         void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && y && rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0,
                 "tc_gelu2d: bad arguments");
    tc_host::launch(gelu2d_kernel, dim3(grid_for(rows * (cols / 8), 256, 16 * sm_count())), dim3(256), 0, stream, 1,
                    reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<__half*>(y), ldy, rows, cols);
    count_launch();
    TC_CHECK_LAUNCH("gelu2d_kernel");
    return TC_OK;
}

extern "C" int tc_time_embed(const float* t, int B, int dim, const void* w1, const float* b1, const void* w2,
                             const float* b2, int hidden, float* out, int accumulate, float* ws, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(t && w1 && w2 && out && ws && B > 0, "tc_time_embed: bad arguments");
    TC_CHECK_ARG(dim % 8 == 0 && hidden % 8 == 0, "tc_time_embed: dim and hidden must be multiples of 8");
    float* emb = ws;                        // [B][dim]
    float* h1 = ws + (long long)B * dim;    // [B][hidden]
    tc_host::launch(sincos_kernel, dim3((B * (dim / 2) + 127) / 128), dim3(128), 0, stream, 1, t, B, dim, emb);
    count_launch();
    TC_CHECK_LAUNCH("sincos_kernel");
    const int blocks = (hidden * 32 + 255) / 256;
    tc_host::launch(small_linear_kernel<float>, dim3(blocks), dim3(256), 0, stream, 1, emb, B, dim, reinterpret_cast<const __half*>(w1), b1,
                                                           hidden, h1, hidden, 0, 0);
    count_launch();
    TC_CHECK_LAUNCH("small_linear_kernel(1)");
    tc_host::launch(small_linear_kernel<float>, dim3(blocks), dim3(256), 0, stream, 1, h1, B, hidden, reinterpret_cast<const __half*>(w2), b2,
                                                           hidden, out, hidden, 1, accumulate);
    count_launch();
    TC_CHECK_LAUNCH("small_linear_kernel(2)");
    return TC_OK;
}

extern "C" int tc_small_linear(const float* x, int B, int K, const void* w, const float* bias, int J, void* y,
                               long long ldy, int silu_in, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x && w && y && B > 0 && K > 0 && K % 8 == 0 && J > 0, "tc_small_linear: bad arguments");
    const int blocks = (int)(((long long)J * 32 + 255) / 256);
    tc_host::launch(small_linear_kernel<__half>, dim3(blocks), dim3(256), 0, stream, 1, x, B, K, reinterpret_cast<const __half*>(w), bias, J,
                                                            reinterpret_cast<__half*>(y), ldy, silu_in, 0);
    count_launch();
    TC_CHECK_LAUNCH("small_linear_kernel");
    return TC_OK;
}

extern "C" int tc_video_u8(const void* x16, const void* x14, int T, int H, int W, int f_begin, int f_end, void* out,
                           void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    TC_CHECK_ARG(x16 && out && T > 0 && H > 0 && W > 0, "tc_video_u8: bad arguments");
    TC_CHECK_ARG(0 <= f_begin && f_begin < f_end && f_end <= T, "tc_video_u8: frame window must satisfy 0 <= f_begin < f_end <= T");
    TC_CHECK_ARG(!x14 || (T >= 4 && T % 2 == 0), "tc_video_u8: the middle-frame splice needs an even T >= 4");
    const long long HW = (long long)H * W;
    const int vec = HW % 8 == 0 && (reinterpret_cast<uintptr_t>(x16) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(x14) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0;
    const long long total = (HW + 7) / 8 * (f_end - f_begin);
    tc_host::launch(video_u8_kernel, dim3(grid_for(total, 256, 16 * sm_count())), dim3(256), 0, stream, 1,
                    reinterpret_cast<const __half*>(x16), reinterpret_cast<const __half*>(x14), T, HW, f_begin,
                    f_end - f_begin, reinterpret_cast<uint8_t*>(out), vec);
    count_launch();
    TC_CHECK_LAUNCH("video_u8_kernel");
    return TC_OK;
}

extern "C" int tc_q_sample(float* x, const float* x0, const float* noise, const float* mask, const float* coef,
                           int clean, int B, long long n, void* stream_v) {
    TC_CHECK_ARG(x && x0 && B > 0 && B <= 65535 && n > 0 && (clean || (noise && coef)), "tc_q_sample: bad arguments");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    const int g = grid_for(n, 256, (4 * sm_count() + B - 1) / B);
    tc_host::launch(q_sample_kernel, dim3(g, B), dim3(256), 0, stream, 1, x, x0, noise, mask, coef, clean ? 1 : 0, n);
    count_launch();
    TC_CHECK_LAUNCH("q_sample_kernel");
    return TC_OK;
}

static int ddim_step_impl(const void* e_c, const void* e_uc, const void* e_img, const float* x, const float* noise,
                          const float* prev_pred_x0, float* x_prev, float* pred_x0, const float* coef, int B,
                          long long n, double* ws, cudaStream_t stream) {
    const __half* ei = reinterpret_cast<const __half*>(e_img);
    tc_host::launch(ddim_reduce_kernel, dim3(dim3(TC_DDIM_PARTIALS, B)), dim3(256), 0, stream, 1,
                    reinterpret_cast<const __half*>(e_c), reinterpret_cast<const __half*>(e_uc), ei, coef, n, ws);
    count_launch();
    TC_CHECK_LAUNCH("ddim_reduce_kernel");
    int g = grid_for(n, 256, 4 * sm_count());
    tc_host::launch(prev_pred_x0 ? ddim_update_kernel<true> : ddim_update_kernel<false>, dim3(dim3(g, B)), dim3(256), 0,
                    stream, 1, reinterpret_cast<const __half*>(e_c), reinterpret_cast<const __half*>(e_uc), ei, x, noise,
                    x_prev, pred_x0, coef, n, ws, TC_DDIM_PARTIALS, prev_pred_x0);
    count_launch();
    TC_CHECK_LAUNCH("ddim_update_kernel");
    return TC_OK;
}

extern "C" int tc_ddim_step(const void* e_c, const void* e_uc, const float* x, const float* noise, float* x_prev,
                            float* pred_x0, const float* coef, int B, long long n, double* ws, void* stream_v) {
    TC_CHECK_ARG(e_c && e_uc && x && noise && x_prev && pred_x0 && coef && ws && B > 0 && n > 1,
                 "tc_ddim_step: bad arguments");
    return ddim_step_impl(e_c, e_uc, nullptr, x, noise, nullptr, x_prev, pred_x0, coef, B, n, ws,
                          reinterpret_cast<cudaStream_t>(stream_v));
}

extern "C" int tc_ddim_step3(const void* e_c, const void* e_uc, const void* e_img, const float* x, const float* noise,
                             float* x_prev, float* pred_x0, const float* coef, int B, long long n, double* ws,
                             void* stream_v) {
    TC_CHECK_ARG(e_c && e_uc && e_img && x && noise && x_prev && pred_x0 && coef && ws && B > 0 && n > 1,
                 "tc_ddim_step3: bad arguments");
    return ddim_step_impl(e_c, e_uc, e_img, x, noise, nullptr, x_prev, pred_x0, coef, B, n, ws,
                          reinterpret_cast<cudaStream_t>(stream_v));
}

extern "C" int tc_dpm_step(const void* e_c, const void* e_uc, const float* x, const float* noise,
                           const float* prev_pred_x0, float* x_prev, float* pred_x0, const float* coef, int B,
                           long long n, double* ws, void* stream_v) {
    TC_CHECK_ARG(e_c && e_uc && x && noise && prev_pred_x0 && x_prev && pred_x0 && coef && ws && B > 0 && n > 1 &&
                 prev_pred_x0 != pred_x0, "tc_dpm_step: bad arguments");
    return ddim_step_impl(e_c, e_uc, nullptr, x, noise, prev_pred_x0, x_prev, pred_x0, coef, B, n, ws,
                          reinterpret_cast<cudaStream_t>(stream_v));
}

extern "C" int tc_dpm_step3(const void* e_c, const void* e_uc, const void* e_img, const float* x, const float* noise,
                            const float* prev_pred_x0, float* x_prev, float* pred_x0, const float* coef, int B,
                            long long n, double* ws, void* stream_v) {
    TC_CHECK_ARG(e_c && e_uc && e_img && x && noise && prev_pred_x0 && x_prev && pred_x0 && coef && ws && B > 0 &&
                 n > 1 && prev_pred_x0 != pred_x0, "tc_dpm_step3: bad arguments");
    return ddim_step_impl(e_c, e_uc, e_img, x, noise, prev_pred_x0, x_prev, pred_x0, coef, B, n, ws,
                          reinterpret_cast<cudaStream_t>(stream_v));
}
