// michigan_b200 — backward-pass CUDA-core kernels (HBM-bound elementwise / reduction / thin-conv
// gradients).  The two big gradient GEMMs live in mg_igemm.cu (data gradient = implicit GEMM on dY with
// flipped sub-kernels) and mg_wgrad.cu (weight gradient, MN-major operands).
//
// Backward identities (SURVEY.md Appendix B), h = act(p), p = xhat*(1+gamma)+beta, xhat = x*ns+nh:
//   dp = dh*act'(p);  dgamma = dp*xhat;  dbeta = dp;  dxhat = dp*(1+gamma)
//   BN:  dx = ns*(dxhat - mean(dxhat) - xhat*mean(dxhat*xhat))   (means over the global N,h,w)
//   IN:  same per (n,c) with g = dy*act'(xhat)
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdlib>
#include <cmath>
#include "mg_internal.h"

namespace mg {

__device__ __forceinline__ float rtf32b(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ float dact(float y, int act) {  // derivative from the OUTPUT sign (relu / lrelu)
    if (act == MG_ACT_RELU) return y > 0.f ? 1.f : 0.f;
    if (act == MG_ACT_LRELU) return y > 0.f ? 1.f : 0.2f;
    return 1.f;
}
static inline int cdivb(long long a, long long b) { return (int)((a + b - 1) / b); }
static int ew_grid_b(long long total, int block = 256) {
    long long g = (total + block - 1) / block;
    const long long cap = (long long)num_sms() * 16;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// block-level reduction of per-thread float4 partials that share a channel group:
// threads are laid out [rows][tpr] (tpr = threads per pixel row = C/4 groups), result atomically added (double).
__device__ __forceinline__ void reduce_rows_atomic(const float (&a)[4], const float (&b)[4], int tpr, int rows, int tr, int tc,
                                                   int g0, int C, double* __restrict__ dst_a, double* __restrict__ dst_b,
                                                   float* sh) {
    // sh: [256][8]
#pragma unroll
    for (int i = 0; i < 4; ++i) { sh[threadIdx.x * 8 + i] = a[i]; sh[threadIdx.x * 8 + 4 + i] = b[i]; }
    __syncthreads();
    if (tr == 0 && threadIdx.x < rows * tpr) {
        double s[4], q[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { s[i] = 0; q[i] = 0; }
        for (int r = 0; r < rows; ++r)
#pragma unroll
            for (int i = 0; i < 4; ++i) { s[i] += sh[(r * tpr + tc) * 8 + i]; q[i] += sh[(r * tpr + tc) * 8 + 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i) { atomicAdd(dst_a + g0 * 4 + i, s[i]); atomicAdd(dst_b + g0 * 4 + i, q[i]); }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------ SPADE backward (elementwise part)
// dh, h, g1: [P][C]; x: [N][hs][ws][C] with P = N*(hs<<xs)*(ws<<xs).  Writes dgb [P][2C] in the packed
// gamma|beta order of the forward operand (per BN-row tile), dxhat [P][C], and adds to sums [2][C] (double).
__global__ void __launch_bounds__(256)
spade_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ hval, const float* __restrict__ g1,
                 const float* __restrict__ x, int xs, int N, int h, int w, int C, const float* __restrict__ ns,
                 const float* __restrict__ nh, int act, int BN, float* __restrict__ dgb, float* __restrict__ dxhat,
                 double* __restrict__ sums, int blocks_total, uint16_t* __restrict__ dgb16, double* __restrict__ bsums) {
    __shared__ float sh[256 * 8];
    const int G = C / 4;
    const int tpr = G < 256 ? G : 256;
    const int rows = 256 / tpr;
    const int tr = threadIdx.x / tpr, tc = threadIdx.x % tpr;
    const long long P = (long long)N * h * w;
    const int hs = h >> xs, ws = w >> xs;
    const int half = BN / 2;
    for (int g0 = tc; g0 < G; g0 += tpr) {
        float a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
        float sg[4] = {0, 0, 0, 0}, sb[4] = {0, 0, 0, 0};     // per-channel sums of dgamma, dbeta (the bias gradients)
        const int c0 = g0 * 4;
        float4 sc = make_float4(0, 0, 0, 0), sf = sc;
        if (threadIdx.x < rows * tpr) {
            sc = __ldg(reinterpret_cast<const float4*>(ns) + g0);
            sf = __ldg(reinterpret_cast<const float4*>(nh) + g0);
            const int tile = c0 / half, r = c0 % half;
            const size_t col_g = (size_t)tile * BN + r, col_b = col_g + half;
            for (long long p = (long long)blockIdx.x * rows + tr; p < P; p += (long long)blocks_total * rows) {
                const int ow = p % w;
                const int oh = (p / w) % h;
                const int n = p / ((long long)w * h);
                const float4 d = __ldg(reinterpret_cast<const float4*>(dh + p * C) + g0);
                const float4 hv = __ldg(reinterpret_cast<const float4*>(hval + p * C) + g0);
                const float4 gg = __ldg(reinterpret_cast<const float4*>(g1 + p * C) + g0);
                const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * hs + (oh >> xs)) * ws + (ow >> xs)) * C) + g0);
                const float dp[4] = {d.x * dact(hv.x, act), d.y * dact(hv.y, act), d.z * dact(hv.z, act), d.w * dact(hv.w, act)};
                const float xh[4] = {fmaf(xv.x, sc.x, sf.x), fmaf(xv.y, sc.y, sf.y), fmaf(xv.z, sc.z, sf.z), fmaf(xv.w, sc.w, sf.w)};
                const float gv[4] = {gg.x, gg.y, gg.z, gg.w};
                float dg[4], dxh[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    dg[i] = dp[i] * xh[i];
                    dxh[i] = dp[i] * gv[i];
                    a[i] += dxh[i];
                    b[i] = fmaf(dxh[i], xh[i], b[i]);
                    sg[i] += dg[i];
                    sb[i] += dp[i];
                }
                if (dgb16) {
                    // bf16 operand of the two gamma|beta gradient GEMMs (their only consumers)
                    const __nv_bfloat162 g01 = __floats2bfloat162_rn(dg[0], dg[1]), g23 = __floats2bfloat162_rn(dg[2], dg[3]);
                    const __nv_bfloat162 b01 = __floats2bfloat162_rn(dp[0], dp[1]), b23 = __floats2bfloat162_rn(dp[2], dp[3]);
                    *reinterpret_cast<uint2*>(dgb16 + p * 2 * C + col_g) = make_uint2(*reinterpret_cast<const uint32_t*>(&g01), *reinterpret_cast<const uint32_t*>(&g23));
                    *reinterpret_cast<uint2*>(dgb16 + p * 2 * C + col_b) = make_uint2(*reinterpret_cast<const uint32_t*>(&b01), *reinterpret_cast<const uint32_t*>(&b23));
                } else {
                    *reinterpret_cast<float4*>(dgb + p * 2 * C + col_g) = make_float4(rtf32b(dg[0]), rtf32b(dg[1]), rtf32b(dg[2]), rtf32b(dg[3]));
                    *reinterpret_cast<float4*>(dgb + p * 2 * C + col_b) = make_float4(rtf32b(dp[0]), rtf32b(dp[1]), rtf32b(dp[2]), rtf32b(dp[3]));
                }
                *reinterpret_cast<float4*>(dxhat + p * C + c0) = make_float4(dxh[0], dxh[1], dxh[2], dxh[3]);
            }
        }
        reduce_rows_atomic(a, b, tpr, rows, tr, tc, g0, C, sums, sums + C, sh);
        if (bsums) reduce_rows_atomic(sg, sb, tpr, rows, tr, tc, g0, C, bsums, bsums + C, sh);
    }
}

// dx_src[n,i,j,c] (+)= scale[c] * sum_{children} (g[child] - m1[c] - xhat*m2[c]),  xhat = x_src*ns + nh.
// scale == null -> 1, m1/m2 == null -> 0 (plain sum over the 2^xs x 2^xs children: upsample backward).
__global__ void bn_bwd_apply_kernel(const float* __restrict__ g, const float* __restrict__ x, int xs, int N, int hs, int ws,
                                    int C, const float* __restrict__ ns, const float* __restrict__ nh,
                                    const double* __restrict__ sums, double inv_count, float* __restrict__ dx,
                                    int accumulate) {
    const int G = C / 4;
    const long long total = (long long)N * hs * ws * G;
    const int f = 1 << xs;
    const int w = ws << xs, h = hs << xs;
    if (sums && inv_count <= 0.0) inv_count = 1.0 / sums[2 * C];   // all-reduced sample count (see bn_finalize_kernel)
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g0 = idx % G;
        long long t = idx / G;
        const int j = t % ws; t /= ws;
        const int i = t % hs;
        const int n = t / hs;
        float sc[4] = {1, 1, 1, 1}, m1[4] = {0, 0, 0, 0}, m2[4] = {0, 0, 0, 0}, xh[4] = {0, 0, 0, 0};
        if (sums) {
            const float4 s = __ldg(reinterpret_cast<const float4*>(ns) + g0);
            const float4 sfh = __ldg(reinterpret_cast<const float4*>(nh) + g0);
            const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + idx);
            sc[0] = s.x; sc[1] = s.y; sc[2] = s.z; sc[3] = s.w;
            xh[0] = fmaf(xv.x, s.x, sfh.x); xh[1] = fmaf(xv.y, s.y, sfh.y); xh[2] = fmaf(xv.z, s.z, sfh.z); xh[3] = fmaf(xv.w, s.w, sfh.w);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                m1[k] = (float)(sums[g0 * 4 + k] * inv_count);
                m2[k] = (float)(sums[C + g0 * 4 + k] * inv_count);
            }
        }
        float acc[4] = {0, 0, 0, 0};
        for (int di = 0; di < f; ++di)
            for (int dj = 0; dj < f; ++dj) {
                const size_t p = ((size_t)n * h + (size_t)i * f + di) * w + (size_t)j * f + dj;
                const float4 v = __ldg(reinterpret_cast<const float4*>(g + p * C) + g0);
                acc[0] += v.x - m1[0] - xh[0] * m2[0];
                acc[1] += v.y - m1[1] - xh[1] * m2[1];
                acc[2] += v.z - m1[2] - xh[2] * m2[2];
                acc[3] += v.w - m1[3] - xh[3] * m2[3];
            }
        float4 o = make_float4(acc[0] * sc[0], acc[1] * sc[1], acc[2] * sc[2], acc[3] * sc[3]);
        if (accumulate) {
            const float4 old = reinterpret_cast<float4*>(dx)[idx];
            o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
        }
        reinterpret_cast<float4*>(dx)[idx] = o;
    }
}

// blend backward (generator.py:186): out = bf*(1-hair) + y*(1-back)
__global__ void blend_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ hair, const float* __restrict__ back,
                                 int N, int h, int w, int C, int ms, int MH, int MW, float* __restrict__ dy,
                                 float* __restrict__ dbf, int acc_bf) {
    const int G = C / 4;
    const long long total = (long long)N * h * w * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long p = idx / G;
        const int ow = p % w;
        const int oh = (p / w) % h;
        const int n = p / ((long long)w * h);
        const size_t mp = ((size_t)n * MH + (size_t)oh * ms) * MW + (size_t)ow * ms;
        const float oh_ = 1.f - __ldg(hair + mp), ob = 1.f - __ldg(back + mp);
        const float4 d = __ldg(reinterpret_cast<const float4*>(dout) + idx);
        reinterpret_cast<float4*>(dy)[idx] = make_float4(d.x * ob, d.y * ob, d.z * ob, d.w * ob);
        float4 b = make_float4(d.x * oh_, d.y * oh_, d.z * oh_, d.w * oh_);
        if (acc_bf) {
            const float4 o = reinterpret_cast<float4*>(dbf)[idx];
            b.x += o.x; b.y += o.y; b.z += o.z; b.w += o.w;
        }
        reinterpret_cast<float4*>(dbf)[idx] = b;
    }
}

// dz = dy * act'(y) * pm1[pix] * pm2[pix]  (y = forward OUTPUT), optional tf32 rounding, optional += into dz
__global__ void act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dz, long long P,
                               int C, int act, const float* __restrict__ pm1, const float* __restrict__ pm2, int round_) {
    const int G = C / 4;
    const long long total = P * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long p = idx / G;
        float m = 1.f;
        if (pm1) m *= __ldg(pm1 + p);
        if (pm2) m *= __ldg(pm2 + p);
        const float4 d = __ldg(reinterpret_cast<const float4*>(dy) + idx);
        float4 yv = make_float4(1.f, 1.f, 1.f, 1.f);
        if (y) yv = __ldg(reinterpret_cast<const float4*>(y) + idx);
        float r[4] = {d.x * dact(yv.x, act) * m, d.y * dact(yv.y, act) * m, d.z * dact(yv.z, act) * m, d.w * dact(yv.w, act) * m};
        if (round_) {
#pragma unroll
            for (int i = 0; i < 4; ++i) r[i] = rtf32b(r[i]);
        }
        reinterpret_cast<float4*>(dz)[idx] = make_float4(r[0], r[1], r[2], r[3]);
    }
}

// ------------------------------------------------------------------------------------ InstanceNorm (+act, +mask) backward
// f = act(xhat)*pm, xhat = x*rstd + shift (ss [N][2][C]).  g = df*pm*act'(xhat).
__global__ void __launch_bounds__(256)
in_bwd_stats_kernel(const float* __restrict__ df, const float* __restrict__ x, const float* __restrict__ ss, long long HW, int C,
                    int act, const float* __restrict__ pm, double* __restrict__ sums, int blocks_per_n) {
    __shared__ float sh[256 * 8];
    const int G = C / 4;
    const int tpr = G < 256 ? G : 256;
    const int rows = 256 / tpr;
    const int n = blockIdx.x / blocks_per_n, blk = blockIdx.x % blocks_per_n;
    const int tr = threadIdx.x / tpr, tc = threadIdx.x % tpr;
    const float* sb = ss + (size_t)n * 2 * C;
    double* out = sums + (size_t)n * 2 * C;
    for (int g0 = tc; g0 < G; g0 += tpr) {
        float a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
        if (threadIdx.x < rows * tpr) {
            const float4 sc = __ldg(reinterpret_cast<const float4*>(sb) + g0);
            const float4 sf = __ldg(reinterpret_cast<const float4*>(sb + C) + g0);
            for (long long p = (long long)blk * rows + tr; p < HW; p += (long long)blocks_per_n * rows) {
                const size_t e = ((size_t)n * HW + p) * C;
                const float4 d = __ldg(reinterpret_cast<const float4*>(df + e) + g0);
                const float4 xv = __ldg(reinterpret_cast<const float4*>(x + e) + g0);
                const float m = pm ? __ldg(pm + (size_t)n * HW + p) : 1.f;
                const float xh[4] = {fmaf(xv.x, sc.x, sf.x), fmaf(xv.y, sc.y, sf.y), fmaf(xv.z, sc.z, sf.z), fmaf(xv.w, sc.w, sf.w)};
                const float dd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float g = dd[i] * m * dact(xh[i], act);
                    a[i] += g;
                    b[i] = fmaf(g, xh[i], b[i]);
                }
            }
        }
        reduce_rows_atomic(a, b, tpr, rows, tr, tc, g0, C, out, out + C, sh);
    }
}
__global__ void in_bwd_apply_kernel(const float* __restrict__ df, const float* __restrict__ x, const float* __restrict__ ss,
                                    const double* __restrict__ sums, int N, long long HW, int C, int act,
                                    const float* __restrict__ pm, float* __restrict__ dx, int round_) {
    const int G = C / 4;
    const long long total = (long long)N * HW * G;
    const double inv = 1.0 / (double)HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g0 = idx % G;
        const long long pix = idx / G;
        const int n = pix / HW;
        const float* sb = ss + (size_t)n * 2 * C;
        const double* sm = sums + (size_t)n * 2 * C;
        const float4 sc = __ldg(reinterpret_cast<const float4*>(sb) + g0);
        const float4 sf = __ldg(reinterpret_cast<const float4*>(sb + C) + g0);
        const float4 d = __ldg(reinterpret_cast<const float4*>(df) + idx);
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + idx);
        const float m = pm ? __ldg(pm + pix) : 1.f;
        const float xh[4] = {fmaf(xv.x, sc.x, sf.x), fmaf(xv.y, sc.y, sf.y), fmaf(xv.z, sc.z, sf.z), fmaf(xv.w, sc.w, sf.w)};
        const float dd[4] = {d.x, d.y, d.z, d.w};
        const float rs[4] = {sc.x, sc.y, sc.z, sc.w};
        float r[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float g = dd[i] * m * dact(xh[i], act);
            const float m1 = (float)(sm[g0 * 4 + i] * inv), m2 = (float)(sm[C + g0 * 4 + i] * inv);
            r[i] = rs[i] * (g - m1 - xh[i] * m2);
            if (round_) r[i] = rtf32b(r[i]);
        }
        reinterpret_cast<float4*>(dx)[idx] = make_float4(r[0], r[1], r[2], r[3]);
    }
}

// ------------------------------------------------------------------------------------ thin conv gradients
// weight gradient of a thin conv: dwt[tap][ci][co] += sum_pix x[pix*s - pad + tap][ci] * dz[pix][co]
// block: 8 output rows x 16 cols tile (same tiling as the forward), thread (co, part) accumulates a slice of taps.
__global__ void __launch_bounds__(256)
thin_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dz, double* __restrict__ dwt, int N, int H, int W,
                  int CinP, int OH, int OW, int Cout, int KH, int KW, int s, int pad, int pad_mode, int R, int tiles_w,
                  int tiles_h, int num_tiles) {
    extern __shared__ __align__(16) float sm[];
    const int PH = 7 * s + KH, PW = 15 * s + KW;
    float* in_s = sm;                        // [PH][PW][CinP]
    float* dz_s = sm + PH * PW * CinP;       // [128][Cout]
    const int K = KH * KW * CinP;
    const int parts = 256 / Cout;            // thread (co, part)
    const int co = threadIdx.x % Cout, part = threadIdx.x / Cout;
    const int kper = (K + parts - 1) / parts;
    const int k0 = part * kper, k1 = min(K, k0 + kper);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tw = tile % tiles_w;
        const int th = (tile / tiles_w) % tiles_h;
        const int n = tile / (tiles_w * tiles_h);
        const int oh0 = th * 8, ow0 = tw * 16;
        const int ih0 = oh0 * s - pad, iw0 = ow0 * s - pad;
        __syncthreads();
        for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
            const int py = i / PW, px = i - py * PW;
            int ih = ih0 + py, iw = iw0 + px;
            if (pad_mode == 1) {
                if (ih < 0) ih = -ih;
                if (ih >= H) ih = 2 * H - 2 - ih;
                if (iw < 0) iw = -iw;
                if (iw >= W) iw = 2 * W - 2 - iw;
            }
            const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
            for (int c = 0; c < CinP; c += 4) {
                float4 v = make_float4(0, 0, 0, 0);
                if (ok) v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H * R + (size_t)ih * R) * ((size_t)W * R) + (size_t)iw * R) * CinP + c));
                *reinterpret_cast<float4*>(in_s + (size_t)i * CinP + c) = v;
            }
        }
        for (int i = threadIdx.x; i < 128 * Cout; i += blockDim.x) {
            const int c = i % Cout, pp = i / Cout;
            const int oh = oh0 + pp / 16, ow = ow0 + pp % 16;
            dz_s[i] = (oh < OH && ow < OW) ? dz[(((size_t)n * OH + oh) * OW + ow) * Cout + c] : 0.f;
        }
        __syncthreads();
        if (part < parts) {
            for (int pp = 0; pp < 128; ++pp) {
                const float d = dz_s[pp * Cout + co];
                const int py = (pp / 16) * s, px = (pp % 16) * s;
#pragma unroll 4
                for (int k = k0; k < k1; ++k) {
                    const int ci = k % CinP, tap = k / CinP;
                    const int kh = tap / KW, kw = tap - kh * KW;
                    acc[k - k0] = fmaf(in_s[((py + kh) * PW + px + kw) * CinP + ci], d, acc[k - k0]);
                }
            }
        }
    }
    if (part < parts)
        for (int k = k0; k < k1; ++k) atomicAdd(dwt + (size_t)k * Cout + co, (double)acc[k - k0]);
}

// Register-tiled weight gradient of a thin conv.  Thread = (group of 4 output
// channels) x (KPT of the KH*KW*CinP weight columns): per pixel one float4 of dz and KPT input values from shared memory
// feed 4*KPT FMAs; the per-CTA partial sums stay in registers across all its tiles and are added at the end into the fp64
// accumulator of the launcher (acc64_*: the result does not depend on the order in which CTAs finish).
template <int KPT>
__global__ void __launch_bounds__(256)
thin_wgrad2_kernel(const float* __restrict__ x, const float* __restrict__ dz, double* __restrict__ dwt, int N, int H, int W,
                   int CinP, int OH, int OW, int Cout, int KH, int KW, int s, int pad, int pad_mode, int R, int tiles_w,
                   int tiles_h, int num_tiles, const float* __restrict__ relu_src, double* __restrict__ bias_sums) {
    extern __shared__ __align__(16) float sm[];
    const int PH = 7 * s + KH, PW = 15 * s + KW;
    float* in_s = sm;                                 // [PH][PW][CinP]
    float* dz_s = sm + ((PH * PW * CinP + 3) & ~3);    // [128][Cout]
    const int K = KH * KW * CinP;
    const int G = Cout >> 2;                          // channel groups (16 or 32)
    const int g = threadIdx.x % G, cg = threadIdx.x / G;
    int xoff[KPT];
#pragma unroll
    for (int i = 0; i < KPT; ++i) {
        const int k = cg * KPT + i;
        const int kk = k < K ? k : 0;
        const int ci = kk % CinP, tap = kk / CinP, kh = tap / KW, kw = tap - kh * KW;
        xoff[i] = (kh * PW + kw) * CinP + ci;
    }
    float acc[KPT][4];
#pragma unroll
    for (int i = 0; i < KPT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    // fused ReLU backward + bias gradient (relu_src = the conv's forward output y: dz <- dz * [y > 0]; bias_sums[c] += sum dz):
    // 256 % G == 0, so a thread stages the same channel group for every pixel and keeps its partial sum in registers
    float4 bsum = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tw = tile % tiles_w;
        const int th = (tile / tiles_w) % tiles_h;
        const int n = tile / (tiles_w * tiles_h);
        const int oh0 = th * 8, ow0 = tw * 16;
        const int ih0 = oh0 * s - pad, iw0 = ow0 * s - pad;
        __syncthreads();
        for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
            const int py = i / PW, px = i - py * PW;
            int ih = ih0 + py, iw = iw0 + px;
            if (pad_mode == 1) {
                if (ih < 0) ih = -ih;
                if (ih >= H) ih = 2 * H - 2 - ih;
                if (iw < 0) iw = -iw;
                if (iw >= W) iw = 2 * W - 2 - iw;
            }
            const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
            for (int c = 0; c < CinP; c += 4) {
                float4 v = make_float4(0, 0, 0, 0);
                if (ok) v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H * R + (size_t)ih * R) * ((size_t)W * R) + (size_t)iw * R) * CinP + c));
                *reinterpret_cast<float4*>(in_s + (size_t)i * CinP + c) = v;
            }
        }
        for (int i = threadIdx.x; i < 128 * G; i += blockDim.x) {
            const int c4 = i % G, pp = i / G;
            const int oh = oh0 + (pp >> 4), ow = ow0 + (pp & 15);
            float4 v = make_float4(0, 0, 0, 0);
            if (oh < OH && ow < OW) {
                const size_t off = (((size_t)n * OH + oh) * OW + ow) * Cout + c4 * 4;
                v = __ldg(reinterpret_cast<const float4*>(dz + off));
                if (relu_src) {
                    const float4 y = __ldg(reinterpret_cast<const float4*>(relu_src + off));
                    v.x = y.x > 0.f ? v.x : 0.f; v.y = y.y > 0.f ? v.y : 0.f; v.z = y.z > 0.f ? v.z : 0.f; v.w = y.w > 0.f ? v.w : 0.f;
                }
                bsum.x += v.x; bsum.y += v.y; bsum.z += v.z; bsum.w += v.w;
            }
            *reinterpret_cast<float4*>(dz_s + (size_t)pp * Cout + c4 * 4) = v;
        }
        __syncthreads();
#pragma unroll 2
        for (int pp = 0; pp < 128; ++pp) {
            const float4 d = *reinterpret_cast<const float4*>(dz_s + pp * Cout + g * 4);
            const float* xb = in_s + (((pp >> 4) * s) * PW + (pp & 15) * s) * CinP;
#pragma unroll
            for (int i = 0; i < KPT; ++i) {
                const float xv = xb[xoff[i]];
                acc[i][0] = fmaf(xv, d.x, acc[i][0]);
                acc[i][1] = fmaf(xv, d.y, acc[i][1]);
                acc[i][2] = fmaf(xv, d.z, acc[i][2]);
                acc[i][3] = fmaf(xv, d.w, acc[i][3]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < KPT; ++i) {
        const int k = cg * KPT + i;
        if (k < K) {
            double* dst = dwt + (size_t)k * Cout + g * 4;
            atomicAdd(dst, (double)acc[i][0]); atomicAdd(dst + 1, (double)acc[i][1]);
            atomicAdd(dst + 2, (double)acc[i][2]); atomicAdd(dst + 3, (double)acc[i][3]);
        }
    }
    if (bias_sums && (256 % G) == 0) {
        const int c4 = threadIdx.x % G;
        atomicAdd(bias_sums + c4 * 4, (double)bsum.x); atomicAdd(bias_sums + c4 * 4 + 1, (double)bsum.y);
        atomicAdd(bias_sums + c4 * 4 + 2, (double)bsum.z); atomicAdd(bias_sums + c4 * 4 + 3, (double)bsum.w);
    }
}

// data gradient of a thin conv restricted to input channels [c_lo, c_lo+3): dimg NCHW [N,3,H,W]
__global__ void __launch_bounds__(256)
thin_dgrad3_kernel(const float* __restrict__ dz, const float* __restrict__ wt, float* __restrict__ dimg, int N, int H, int W,
                   int CinP, int OH, int OW, int Cout, int KH, int KW, int s, int pad, int c_lo) {
    extern __shared__ __align__(16) float w_s[];   // [KH*KW][3][Cout]
    for (int i = threadIdx.x; i < KH * KW * 3 * Cout; i += blockDim.x) {
        const int co = i % Cout, c = (i / Cout) % 3, tap = i / (3 * Cout);
        w_s[i] = wt[((size_t)tap * CinP + c_lo + c) * Cout + co];
    }
    __syncthreads();
    const long long total = (long long)N * H * W;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int iw = idx % W;
        const int ih = (idx / W) % H;
        const int n = idx / ((long long)W * H);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int kh = 0; kh < KH; ++kh) {
            const int t = ih + pad - kh;
            if (t < 0 || t % s != 0) continue;
            const int oh = t / s;
            if (oh >= OH) continue;
            for (int kw = 0; kw < KW; ++kw) {
                const int u = iw + pad - kw;
                if (u < 0 || u % s != 0) continue;
                const int ow = u / s;
                if (ow >= OW) continue;
                const float4* dp = reinterpret_cast<const float4*>(dz + (((size_t)n * OH + oh) * OW + ow) * Cout);
                const float* wp = w_s + (size_t)(kh * KW + kw) * 3 * Cout;
                for (int c4 = 0; c4 < Cout / 4; ++c4) {
                    const float4 d = __ldg(dp + c4);
                    const float4 w0 = *reinterpret_cast<const float4*>(wp + c4 * 4);
                    const float4 w1 = *reinterpret_cast<const float4*>(wp + Cout + c4 * 4);
                    const float4 w2 = *reinterpret_cast<const float4*>(wp + 2 * Cout + c4 * 4);
                    a0 += d.x * w0.x + d.y * w0.y + d.z * w0.z + d.w * w0.w;
                    a1 += d.x * w1.x + d.y * w1.y + d.z * w1.z + d.w * w1.w;
                    a2 += d.x * w2.x + d.y * w2.y + d.z * w2.z + d.w * w2.w;
                }
            }
        }
        const size_t hw = (size_t)H * W, o = (size_t)n * 3 * hw + (size_t)ih * W + iw;
        dimg[o] += a0; dimg[o + hw] += a1; dimg[o + 2 * hw] += a2;
    }
}

// ------------------------------------------------------------------------------------ conv_img backward
// y = tanh(conv3x3(lrelu(x)) + b): dz = dy*(1-y^2) [N,3,H,W -> NHWC4]; dx = lrelu'(x) * conv_T(dz, W)
__global__ void conv_img_dz_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dz4, int N,
                                   int Cout, long long HW, int act_out) {
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int n = idx / HW;
        const long long p = idx - (long long)n * HW;
        float r[4] = {0, 0, 0, 0};
        for (int c = 0; c < Cout; ++c) {
            const size_t o = ((size_t)n * Cout + c) * HW + p;
            const float yy = y[o];
            r[c] = dy[o] * (act_out == MG_ACT_TANH ? (1.f - yy * yy) : 1.f);
        }
        reinterpret_cast<float4*>(dz4)[idx] = make_float4(r[0], r[1], r[2], r[3]);
    }
}
__global__ void __launch_bounds__(256)
conv_img_dgrad_kernel(const float* __restrict__ dz4, const float* __restrict__ x, const float* __restrict__ w,
                      float* __restrict__ dx, int N, int H, int W, int Cin, int Cout, int act_in) {
    extern __shared__ __align__(16) float w_s[];  // [9][4(co)][Cin]
    for (int i = threadIdx.x; i < 9 * 4 * Cin; i += blockDim.x) {
        const int ci = i % Cin, co = (i / Cin) & 3, tap = i / (4 * Cin);
        w_s[i] = co < Cout ? w[((size_t)co * Cin + ci) * 9 + tap] : 0.f;
    }
    __syncthreads();
    const int G = Cin / 4;
    const long long total = (long long)N * H * W * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g0 = idx % G;
        const long long pix = idx / G;
        const int iw = pix % W;
        const int ih = (pix / W) % H;
        const int n = pix / ((long long)W * H);
        float a[4] = {0, 0, 0, 0};
        for (int kh = 0; kh < 3; ++kh) {
            const int oh = ih + 1 - kh;
            if (oh < 0 || oh >= H) continue;
            for (int kw = 0; kw < 3; ++kw) {
                const int ow = iw + 1 - kw;
                if (ow < 0 || ow >= W) continue;
                const float4 d = __ldg(reinterpret_cast<const float4*>(dz4) + ((size_t)n * H + oh) * W + ow);
                const float* wp = w_s + (size_t)(kh * 3 + kw) * 4 * Cin + g0 * 4;
                const float dd[3] = {d.x, d.y, d.z};
#pragma unroll
                for (int co = 0; co < 3; ++co) {
                    const float4 wv = *reinterpret_cast<const float4*>(wp + co * Cin);
                    a[0] = fmaf(dd[co], wv.x, a[0]); a[1] = fmaf(dd[co], wv.y, a[1]);
                    a[2] = fmaf(dd[co], wv.z, a[2]); a[3] = fmaf(dd[co], wv.w, a[3]);
                }
            }
        }
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + idx);
        reinterpret_cast<float4*>(dx)[idx] = make_float4(a[0] * dact(xv.x, act_in), a[1] * dact(xv.y, act_in),
                                                         a[2] * dact(xv.z, act_in), a[3] * dact(xv.w, act_in));
    }
}
// dW[co][ci][tap] += sum_pix dz[pix][co] * act(x[pix+tap][ci]); db[co] += sum dz.  One block = 8x32 pixel tile.
__global__ void __launch_bounds__(256)
conv_img_wgrad_kernel(const float* __restrict__ dz4, const float* __restrict__ x, double* __restrict__ dw, double* __restrict__ db,
                      int N, int H, int W, int Cin, int Cout, int act_in, int tiles_w, int tiles_h, int num_tiles) {
    extern __shared__ __align__(16) float sm[];
    const int PW = 34, PH = 10, NP = PW * PH;
    float* in_s = sm;                 // [NP][Cin]  (+1 pad per pixel row to dodge bank conflicts)
    float* dz_s = sm + (size_t)NP * (Cin + 1);   // [256][4]
    // thread -> (ci, tap group): Cin*9 products per co; threads = 256: each handles (ci = t % Cin, taps t/Cin .. step 256/Cin)
    const int ci = threadIdx.x % Cin, tg = threadIdx.x / Cin, tgn = 256 / Cin;
    // taps of this thread: tg, tg + tgn, tg + 2*tgn, ... (at most 5 for Cin <= 128); the accumulators are indexed by the UNROLLED
    // slot j, never by the run-time tap (a run-time index would put the whole array in local memory)
    constexpr int kSlots = 5;
    float acc[kSlots][3];
#pragma unroll
    for (int j = 0; j < kSlots; ++j) acc[j][0] = acc[j][1] = acc[j][2] = 0.f;
    float bacc[3] = {0, 0, 0};
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
        const int h0 = th * 8 - 1, w0 = tw * 32 - 1;
        __syncthreads();
        {
            // fill: thread = (pixel group, float4 channel group); one integer division per pixel instead of four per element
            const int C4 = Cin >> 2, c4 = threadIdx.x % C4, pg = threadIdx.x / C4, npg = 256 / C4;
            for (int pp = pg; pp < NP; pp += npg) {
                const int py = pp / PW, px = pp - py * PW;
                const int ih = h0 + py, iw = w0 + px;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
                    v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H + ih) * W + iw) * Cin) + c4);
                    if (act_in == MG_ACT_LRELU) {
                        v.x = v.x > 0.f ? v.x : 0.2f * v.x; v.y = v.y > 0.f ? v.y : 0.2f * v.y;
                        v.z = v.z > 0.f ? v.z : 0.2f * v.z; v.w = v.w > 0.f ? v.w : 0.2f * v.w;
                    }
                }
                float* d = in_s + (size_t)pp * (Cin + 1) + c4 * 4;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
        }
        {
            const int ly = threadIdx.x >> 5, lx = threadIdx.x & 31;
            const int oh = th * 8 + ly, ow = tw * 32 + lx;
            float4 d = make_float4(0, 0, 0, 0);
            if (oh < H && ow < W) d = __ldg(reinterpret_cast<const float4*>(dz4) + ((size_t)n * H + oh) * W + ow);
            *reinterpret_cast<float4*>(dz_s + threadIdx.x * 4) = d;
            if (tg == 0 && ci < 3) {}
        }
        __syncthreads();
        if (tg < tgn) {
            for (int pp = 0; pp < 256; ++pp) {
                const float4 d = *reinterpret_cast<const float4*>(dz_s + pp * 4);
                const int ly = pp >> 5, lx = pp & 31;
#pragma unroll
                for (int j = 0; j < kSlots; ++j) {
                    const int t = tg + j * tgn;
                    if (t < 9) {
                        const int kh = t / 3, kw = t - kh * 3;
                        const float v = in_s[(size_t)((ly + kh) * PW + lx + kw) * (Cin + 1) + ci];
                        acc[j][0] = fmaf(d.x, v, acc[j][0]); acc[j][1] = fmaf(d.y, v, acc[j][1]); acc[j][2] = fmaf(d.z, v, acc[j][2]);
                    }
                }
            }
        }
        if (threadIdx.x < 32) {
            // bias gradient: lane sums 8 pixels, butterfly over the warp; lanes 0..2 keep channels 0..2
            float s0 = 0.f, s1 = 0.f, s2 = 0.f;
            for (int pp = threadIdx.x; pp < 256; pp += 32) { s0 += dz_s[pp * 4]; s1 += dz_s[pp * 4 + 1]; s2 += dz_s[pp * 4 + 2]; }
            for (int o = 16; o > 0; o >>= 1) {
                s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            }
            if (threadIdx.x == 0) bacc[0] += s0;
            if (threadIdx.x == 1) bacc[1] += s1;
            if (threadIdx.x == 2) bacc[2] += s2;
        }
    }
    if (tg < tgn) {
#pragma unroll
        for (int j = 0; j < kSlots; ++j) {
            const int t = tg + j * tgn;
            if (t < 9) {
#pragma unroll
                for (int co = 0; co < 3; ++co)
                    if (co < Cout) atomicAdd(dw + ((size_t)co * Cin + ci) * 9 + t, (double)acc[j][co]);
            }
        }
    }
    if (threadIdx.x < Cout && db) atomicAdd(db + threadIdx.x, (double)bacc[threadIdx.x]);
}

// ------------------------------------------------------------------------------------ Cin -> 1 conv backward
__global__ void __launch_bounds__(256)
conv_to1_dgrad_kernel(const float* __restrict__ dl, const float* __restrict__ w, float* __restrict__ dx, int N,
                      int H, int W, int Cin, int KH, int KW, int pad, int OH, int OW, int accumulate) {
    // weights transposed to [tap][Cin] in shared memory: consecutive lanes (channel groups) read consecutive float4
    extern __shared__ __align__(16) float w_s[];
    for (int i = threadIdx.x; i < KH * KW * Cin; i += blockDim.x) {
        const int c = i % Cin, tap = i / Cin;
        w_s[i] = w[(size_t)c * KH * KW + tap];
    }
    __syncthreads();
    const int G = Cin / 4;
    const long long total = (long long)N * H * W * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g0 = idx % G;
        const long long pix = idx / G;
        const int iw = pix % W;
        const int ih = (pix / W) % H;
        const int n = pix / ((long long)W * H);
        float a[4] = {0, 0, 0, 0};
        for (int kh = 0; kh < KH; ++kh) {
            const int oh = ih + pad - kh;
            if (oh < 0 || oh >= OH) continue;
            for (int kw = 0; kw < KW; ++kw) {
                const int ow = iw + pad - kw;
                if (ow < 0 || ow >= OW) continue;
                const float d = __ldg(dl + ((size_t)n * OH + oh) * OW + ow);
                const float4 wv = *reinterpret_cast<const float4*>(w_s + (size_t)(kh * KW + kw) * Cin + g0 * 4);
                a[0] = fmaf(d, wv.x, a[0]); a[1] = fmaf(d, wv.y, a[1]); a[2] = fmaf(d, wv.z, a[2]); a[3] = fmaf(d, wv.w, a[3]);
            }
        }
        float4 o = make_float4(a[0], a[1], a[2], a[3]);
        if (accumulate) {
            const float4 old = reinterpret_cast<float4*>(dx)[idx];
            o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
        }
        reinterpret_cast<float4*>(dx)[idx] = o;
    }
}
// dw[ci][tap] += sum_pix dl[pix] * x[pix + tap][ci]; one warp per (tap, 128-channel slab), grid-stride over pixels
__global__ void __launch_bounds__(256)
conv_to1_wgrad_kernel(const float* __restrict__ dl, const float* __restrict__ x, double* __restrict__ dw, double* __restrict__ db,
                      int N, int H, int W, int Cin, int KH, int KW, int pad, int OH, int OW) {
    const int tap = blockIdx.y;
    const int kh = tap / KW, kw = tap - kh * KW;
    const int G = Cin / 4;
    const long long total = (long long)N * OH * OW;
    const int chunk = (int)((total + gridDim.x - 1) / gridDim.x);
    const long long p0 = (long long)blockIdx.x * chunk, p1 = p0 + chunk < total ? p0 + chunk : total;
    for (int g0 = threadIdx.x; g0 < G; g0 += blockDim.x) {
        float a[4] = {0, 0, 0, 0};
        for (long long o = p0; o < p1; ++o) {
            const int ow = o % OW;
            const int oh = (o / OW) % OH;
            const int n = o / ((long long)OW * OH);
            const int ih = oh + kh - pad, iw = ow + kw - pad;
            if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
            const float d = __ldg(dl + o);
            const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H + ih) * W + iw) * Cin) + g0);
            a[0] = fmaf(d, xv.x, a[0]); a[1] = fmaf(d, xv.y, a[1]); a[2] = fmaf(d, xv.z, a[2]); a[3] = fmaf(d, xv.w, a[3]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) atomicAdd(dw + (size_t)(g0 * 4 + i) * KH * KW + tap, (double)a[i]);
    }
    if (tap == 0 && threadIdx.x == 0 && db) {
        float s = 0.f;
        for (long long o = p0; o < p1; ++o) s += dl[o];
        atomicAdd(db, (double)s);
    }
}

// ------------------------------------------------------------------------------------ pooling / resize / pad backward
__global__ void avgpool3s2_bwd_kernel(const float* __restrict__ dout, float* __restrict__ din, int N, int H, int W, int C,
                                      int OH, int OW) {
    const int G = C / 4;
    const long long total = (long long)N * H * W * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g0 = idx % G;
        const long long pix = idx / G;
        const int iw = pix % W;
        const int ih = (pix / W) % H;
        const int n = pix / ((long long)W * H);
        float4 a = make_float4(0, 0, 0, 0);
        for (int oh = (ih - 1 + 1) / 2; oh <= (ih + 1) / 2; ++oh) {
            if (oh < 0 || oh >= OH || abs(oh * 2 - ih) > 1) continue;
            for (int ow = (iw) / 2; ow <= (iw + 1) / 2; ++ow) {
                if (ow < 0 || ow >= OW || abs(ow * 2 - iw) > 1) continue;
                const int ch = min(oh * 2 + 1, H - 1) - max(oh * 2 - 1, 0) + 1;
                const int cw = min(ow * 2 + 1, W - 1) - max(ow * 2 - 1, 0) + 1;
                const float inv = 1.f / (float)(ch * cw);
                const float4 d = __ldg(reinterpret_cast<const float4*>(dout + (((size_t)n * OH + oh) * OW + ow) * C) + g0);
                a.x += d.x * inv; a.y += d.y * inv; a.z += d.z * inv; a.w += d.w * inv;
            }
        }
        float4 o = reinterpret_cast<float4*>(din)[idx];
        o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
        reinterpret_cast<float4*>(din)[idx] = o;
    }
}
// reflect-pad backward: fold the padded gradient [N,H+2p,W+2p,C] back onto [N,H,W,C]
__global__ void reflect_pad_bwd_kernel(const float* __restrict__ dpad, float* __restrict__ dx, int N, int H, int W, int C, int p,
                                       int accumulate) {
    const int G = C / 4;
    const int PH = H + 2 * p, PW = W + 2 * p;
    const long long total = (long long)N * H * W * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g0 = idx % G;
        const long long pix = idx / G;
        const int iw = pix % W;
        const int ih = (pix / W) % H;
        const int n = pix / ((long long)W * H);
        // padded rows that map to ih: ih+p, and the mirror images when within p of a border
        int hs_[3], nh = 0, ws_[3], nw = 0;
        hs_[nh++] = ih + p;
        if (ih >= 1 && ih <= p) hs_[nh++] = p - ih;
        if (ih <= H - 2 && ih >= H - 1 - p) hs_[nh++] = p + 2 * (H - 1) - ih;
        ws_[nw++] = iw + p;
        if (iw >= 1 && iw <= p) ws_[nw++] = p - iw;
        if (iw <= W - 2 && iw >= W - 1 - p) ws_[nw++] = p + 2 * (W - 1) - iw;
        float4 a = make_float4(0, 0, 0, 0);
        for (int i = 0; i < nh; ++i)
            for (int j = 0; j < nw; ++j) {
                const float4 d = __ldg(reinterpret_cast<const float4*>(dpad + (((size_t)n * PH + hs_[i]) * PW + ws_[j]) * C) + g0);
                a.x += d.x; a.y += d.y; a.z += d.z; a.w += d.w;
            }
        if (accumulate) {
            const float4 o = reinterpret_cast<float4*>(dx)[idx];
            a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
        }
        reinterpret_cast<float4*>(dx)[idx] = a;
    }
}
// bilinear (align_corners=False) backward: scatter with fp64 atomics into the launcher's acc64 buffer (tiny tensors:
// reference-encoder tail)
__global__ void resize_bilinear_bwd_kernel(const float* __restrict__ dout, double* __restrict__ din, int N, int H, int W, int C,
                                           int OH, int OW) {
    const long long total = (long long)N * OH * OW * C;
    const float sh = (float)H / OH, sw = (float)W / OW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = idx % C;
        long long t = idx / C;
        const int ow = t % OW; t /= OW;
        const int oh = t % OH;
        const int n = t / OH;
        float fy = ((float)oh + 0.5f) * sh - 0.5f; if (fy < 0.f) fy = 0.f;
        float fx = ((float)ow + 0.5f) * sw - 0.5f; if (fx < 0.f) fx = 0.f;
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
        const float ly = fy - y0, lx = fx - x0, d = dout[idx];
        double* b = din + (size_t)n * H * W * C + c;
        atomicAdd(b + ((size_t)y0 * W + x0) * C, (double)(d * (1.f - ly) * (1.f - lx)));
        atomicAdd(b + ((size_t)y0 * W + x1) * C, (double)(d * (1.f - ly) * lx));
        atomicAdd(b + ((size_t)y1 * W + x0) * C, (double)(d * ly * (1.f - lx)));
        atomicAdd(b + ((size_t)y1 * W + x1) * C, (double)(d * ly * lx));
    }
}
// masked mean broadcast backward: out[p,c] = mean_c * mtag[p], mean_c = sum_q x[q,c]*mref[q] / max(cnt,1)
//  => dx[q,c] = mref[q]/max(cnt,1) * sum_p dout[p,c]*mtag[p]
__global__ void masked_mean_bcast_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ mref,
                                             const float* __restrict__ mtag, float* __restrict__ dx, int N, int h, int w, int C,
                                             int MH, int MW) {
    const int n = blockIdx.y;
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int row = threadIdx.x >> 5;
    const int sh = MH / h, sw = MW / w;
    __shared__ float red[8][33];
    __shared__ float cnt_s[8];
    float acc = 0.f, cnt = 0.f;
    for (int pidx = row; pidx < h * w; pidx += 8) {
        const int ph = pidx / w, pw = pidx - ph * w;
        cnt += mref[((size_t)n * MH + (size_t)ph * sh) * MW + (size_t)pw * sw];
        const float mt = mtag[((size_t)n * MH + (size_t)ph * sh) * MW + (size_t)pw * sw];
        if (c < C) acc += dout[(((size_t)n * h + ph) * w + pw) * C + c] * mt;
    }
    red[row][threadIdx.x & 31] = acc;
    if ((threadIdx.x & 31) == 0) cnt_s[row] = cnt;
    __syncthreads();
    float tot = 0.f, ctot = 0.f;
    for (int r = 0; r < 8; ++r) { tot += red[r][threadIdx.x & 31]; ctot += cnt_s[r]; }
    const float gmean = tot / fmaxf(ctot, 1.f);
    for (int pidx = row; pidx < h * w; pidx += 8) {
        const int ph = pidx / w, pw = pidx - ph * w;
        const float m = mref[((size_t)n * MH + (size_t)ph * sh) * MW + (size_t)pw * sw];
        if (c < C) dx[(((size_t)n * h + ph) * w + pw) * C + c] = gmean * m;
    }
}

// ------------------------------------------------------------------------------------ spectral norm backward
// dW_orig = (dWt - <dWt, Wt> u v^T) / sigma, Wt = W_orig/sigma:  s = sum(dWt*W_orig)*inv_sigma
__global__ void __launch_bounds__(256) sn_bwd_dot_kernel(const float* __restrict__ dwt, const float* __restrict__ w, long long n,
                                                         double* __restrict__ out) {
    double a = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        a += (double)dwt[i] * (double)w[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
    __shared__ double sh[8];
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
        for (int i = 0; i < 8; ++i) s += sh[i];
        atomicAdd(out, s);
    }
}
__global__ void sn_bwd_apply_kernel(const float* __restrict__ dwt, const float* __restrict__ u, const float* __restrict__ v,
                                    const float* __restrict__ inv_sigma, const double* __restrict__ dot, float* __restrict__ dw,
                                    int O, long long K, int accumulate) {
    const long long total = (long long)O * K;
    const float is = *inv_sigma;
    const float s = (float)(*dot) * is;  // <dWt, Wt>
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int o = i / K;
        const long long k = i - (long long)o * K;
        const float r = (dwt[i] - s * u[o] * v[k]) * is;
        dw[i] = accumulate ? dw[i] + r : r;
    }
}

// gamma|beta operand for the data gradient of the SPADE GEMM: out[ci][tap'][R] with R the packed row
// order of the forward operand, taps flipped (3x3, stride 1): out[ci][(2-kh)*3+(2-kw)][R] = W_R[ci][kh][kw]
__global__ void pack_weight_dgrad_gb_kernel(const float* __restrict__ wg, const float* __restrict__ wb, float* __restrict__ out,
                                            int C, int I, int BN) {
    const long long total = (long long)I * 9 * 2 * C;
    const int half = BN / 2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int R = idx % (2 * C);
        long long t = idx / (2 * C);
        const int tap = t % 9;
        const int ci = t / 9;
        const int tile = R / BN, rr = R % BN;
        const float* src = rr < half ? wg : wb;
        const int c = tile * half + (rr < half ? rr : rr - half);
        const int kh = 2 - tap / 3, kw = 2 - tap % 3;
        out[idx] = rtf32b(src[(((long long)c * I + ci) * 3 + kh) * 3 + kw]);
    }
}
// packed [2C][9*I] gamma|beta weight gradient -> the two OIHW gradients (+=)
__global__ void unpack_wgrad_gb_kernel(const float* __restrict__ dwp, float* __restrict__ dwg, float* __restrict__ dwb, int C, int I,
                                       int BN, int accumulate) {
    const long long total = 2LL * C * I * 9;
    const int half = BN / 2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = idx % I;
        long long t = idx / I;
        const int tap = t % 9;
        const int R = t / 9;
        const int tile = R / BN, rr = R % BN;
        float* dst = rr < half ? dwg : dwb;
        const int c = tile * half + (rr < half ? rr : rr - half);
        const size_t o = ((size_t)c * I + i) * 9 + tap;
        dst[o] = accumulate ? dst[o] + dwp[idx] : dwp[idx];
    }
}

}  // namespace mg

using namespace mg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

__global__ void cvt16_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, long long n4, int fmt) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
        uint32_t lo, hi;
        if (fmt == 1) {
            const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
            lo = *reinterpret_cast<const uint32_t*>(&a); hi = *reinterpret_cast<const uint32_t*>(&b);
        } else {
            const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
            lo = *reinterpret_cast<const uint32_t*>(&a); hi = *reinterpret_cast<const uint32_t*>(&b);
        }
        reinterpret_cast<uint2*>(dst)[i] = make_uint2(lo, hi);
    }
}

extern "C" int mg_cvt16(const float* src, void* dst, long long n, int fmt, void* stream) {
    if (!src || !dst) return set_error(-1, "mg_cvt16: null pointer");
    if (n % 4 != 0 || (fmt != 1 && fmt != 2)) return set_error(-2, "mg_cvt16: n %% 4 == 0, fmt 1 | 2");
    cvt16_kernel<<<ew_grid_b(n / 4), 256, 0, ST(stream)>>>(src, static_cast<uint16_t*>(dst), n / 4, fmt);
    return check_launch("mg_cvt16");
}

extern "C" int mg_spade_bwd(const float* dh, const float* h, const float* g1, const float* x, int x_shift, int N, int H, int W, int C,
                            const float* nscale, const float* nshift, int act, int BN, float* dgb, float* dxhat, double* sums,
                            void* dgb16, double* bias_sums, void* stream) {
    if (!dh || !h || !g1 || !x || !nscale || !nshift || (!dgb && !dgb16) || !dxhat || !sums) return set_error(-1, "mg_spade_bwd: null pointer");
    if (C % 4 != 0 || C > 1024 || BN % 64 != 0 || (2 * C) % BN != 0) return set_error(-2, "mg_spade_bwd: bad C/BN");
    const int G = C / 4, tpr = G < 256 ? G : 256, rows = 256 / tpr;
    const long long P = (long long)N * H * W;
    long long blocks = (P + rows * 8 - 1) / (rows * 8);
    const long long cap = (long long)num_sms() * 4;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    spade_bwd_kernel<<<(int)blocks, 256, 0, ST(stream)>>>(dh, h, g1, x, x_shift, N, H, W, C, nscale, nshift, act, BN, dgb, dxhat,
                                                          sums, (int)blocks, static_cast<uint16_t*>(dgb16), bias_sums);
    return check_launch("mg_spade_bwd");
}
extern "C" int mg_bn_bwd_apply(const float* g, const float* x, int x_shift, int N, int hs, int ws, int C, const float* nscale,
                               const float* nshift, const double* sums, double count, float* dx, int accumulate, void* stream) {
    if (!g || !dx) return set_error(-1, "mg_bn_bwd_apply: null pointer");
    if (sums && (!x || !nscale || !nshift)) return set_error(-2, "mg_bn_bwd_apply: sums need x/nscale/nshift");
    bn_bwd_apply_kernel<<<ew_grid_b((long long)N * hs * ws * (C / 4)), 256, 0, ST(stream)>>>(g, x, x_shift, N, hs, ws, C, nscale, nshift,
                                                                                            sums, (sums && count > 0.0) ? 1.0 / count : 0.0, dx, accumulate);
    return check_launch("mg_bn_bwd_apply");
}
extern "C" int mg_blend_bwd(const float* dout, const float* hair, const float* back, int N, int H, int W, int C, int mask_stride,
                            int MH, int MW, float* dy, float* dbf, int accumulate_bf, void* stream) {
    if (!dout || !hair || !back || !dy || !dbf) return set_error(-1, "mg_blend_bwd: null pointer");
    blend_bwd_kernel<<<ew_grid_b((long long)N * H * W * (C / 4)), 256, 0, ST(stream)>>>(dout, hair, back, N, H, W, C, mask_stride, MH, MW,
                                                                                       dy, dbf, accumulate_bf);
    return check_launch("mg_blend_bwd");
}
extern "C" int mg_act_bwd(const float* dy, const float* y, float* dz, long long P, int C, int act, const float* pm1, const float* pm2,
                          int round_tf32, void* stream) {
    if (!dy || !dz) return set_error(-1, "mg_act_bwd: null pointer");
    if (C % 4 != 0) return set_error(-2, "mg_act_bwd: C%%4");
    act_bwd_kernel<<<ew_grid_b(P * (C / 4)), 256, 0, ST(stream)>>>(dy, y, dz, P, C, act, pm1, pm2, round_tf32);
    return check_launch("mg_act_bwd");
}
extern "C" int mg_in_bwd(const float* df, const float* x, const float* ss, double* sums, float* dx, int N, long long HW, int C, int act,
                         const float* pmul, int round_tf32, void* stream) {
    if (!df || !x || !ss || !sums || !dx) return set_error(-1, "mg_in_bwd: null pointer");
    if (C % 4 != 0 || C > 1024) return set_error(-2, "mg_in_bwd: bad C");
    const int G = C / 4, tpr = G < 256 ? G : 256, rows = 256 / tpr;
    long long want = (HW + rows * 8 - 1) / (rows * 8);
    long long cap = ((long long)num_sms() * 4 + N - 1) / N;
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    cudaMemsetAsync(sums, 0, (size_t)N * 2 * C * sizeof(double), ST(stream));
    in_bwd_stats_kernel<<<(int)want * N, 256, 0, ST(stream)>>>(df, x, ss, HW, C, act, pmul, sums, (int)want);
    count_launch();
    in_bwd_apply_kernel<<<ew_grid_b((long long)N * HW * G), 256, 0, ST(stream)>>>(df, x, ss, sums, N, HW, C, act, pmul, dx, round_tf32);
    return check_launch("mg_in_bwd");
}
extern "C" int mg_thin_wgrad(const float* x, const float* dz, float* dwt, int N, int H, int W, int CinP, int OH, int OW, int Cout, int KH,
                             int KW, int stride, int pad, int pad_mode, int seg_resize, const float* relu_src, double* bias_sums,
                             void* stream) {
    if (!x || !dz || !dwt) return set_error(-1, "mg_thin_wgrad: null pointer");
    if (Cout > 256 || 256 % Cout != 0) return set_error(-2, "mg_thin_wgrad: Cout must divide 256");
    const int K = KH * KW * CinP, parts = 256 / Cout;
    const int PH = 7 * stride + KH, PW = 15 * stride + KW;
    const int tiles_w = cdivb(OW, 16), tiles_h = cdivb(OH, 8), num_tiles = tiles_w * tiles_h * N;
    int grid = num_sms();
    if (grid > num_tiles) grid = num_tiles;
    const int R = seg_resize > 0 ? seg_resize : 1;
    double* acc = nullptr;
    int rc = acc64_alloc(&acc, (size_t)K * Cout, ST(stream));
    if (rc) return rc;
    // partial sums -> acc (fp64, order-independent) -> dwt
    auto finish = [&](int rc0) {
        if (!rc0) rc0 = acc64_fold(acc, dwt, (size_t)K * Cout, 0, ST(stream));
        const int rc1 = acc64_free(acc, ST(stream));
        return rc0 ? rc0 : rc1;
    };
    // register-tiled kernel: Cout 64/128, columns per thread = ceil(K / (256 / (Cout/4)))
    const int CG = Cout == 64 || Cout == 128 ? 256 / (Cout / 4) : 0;
    const int kpt = CG ? (K + CG - 1) / CG : 0;
    if (CG && kpt <= 13 && CinP % 4 == 0) {
        const size_t smem = ((((size_t)PH * PW * CinP + 3) & ~(size_t)3) + 128 * (size_t)Cout) * 4;
        // load -> sync -> compute per tile: co-resident CTAs overlap one's loads with another's FMAs
        int per_sm = (int)((200 * 1024) / (smem + 1024));
        if (per_sm > 3) per_sm = 3;
        if (per_sm < 1) per_sm = 1;
        grid = num_sms() * per_sm;
        if (grid > num_tiles) grid = num_tiles;
#define MG_TW2(KP)                                                                                                              \
    do {                                                                                                                         \
        cudaError_t e = cudaFuncSetAttribute(thin_wgrad2_kernel<KP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);     \
        if (e != cudaSuccess) return finish(set_error((int)e, "thin_wgrad2 attr: %s", cudaGetErrorString(e)));                   \
        thin_wgrad2_kernel<KP><<<grid, 256, smem, ST(stream)>>>(x, dz, acc, N, H, W, CinP, OH, OW, Cout, KH, KW, stride, pad,    \
                                                                pad_mode, R, tiles_w, tiles_h, num_tiles, relu_src, bias_sums);   \
    } while (0)
        if (kpt <= 3) MG_TW2(3);
        else if (kpt <= 5) MG_TW2(5);
        else if (kpt <= 8) MG_TW2(8);
        else MG_TW2(13);
#undef MG_TW2
        return finish(check_launch("mg_thin_wgrad"));
    }
    if (relu_src || bias_sums)
        return finish(set_error(-4, "mg_thin_wgrad: the fused ReLU / bias-sum form needs the register-tiled kernel (Cout 64 | 128)"));
    if ((K + parts - 1) / parts > 64) return finish(set_error(-3, "mg_thin_wgrad: K %d too large for %d parts", K, parts));
    const size_t smem = ((size_t)PH * PW * CinP + 128 * (size_t)Cout) * 4;
    cudaError_t e = cudaFuncSetAttribute(thin_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return finish(set_error((int)e, "thin_wgrad attr: %s", cudaGetErrorString(e)));
    int grid2 = num_sms() * 2;
    if (grid2 > num_tiles) grid2 = num_tiles;
    thin_wgrad_kernel<<<grid2, 256, smem, ST(stream)>>>(x, dz, acc, N, H, W, CinP, OH, OW, Cout, KH, KW, stride, pad, pad_mode, R,
                                                        tiles_w, tiles_h, num_tiles);
    return finish(check_launch("mg_thin_wgrad"));
}
extern "C" int mg_thin_dgrad3(const float* dz, const float* wt, float* dimg_nchw, int N, int H, int W, int CinP, int OH, int OW, int Cout,
                              int KH, int KW, int stride, int pad, int c_lo, void* stream) {
    if (!dz || !wt || !dimg_nchw) return set_error(-1, "mg_thin_dgrad3: null pointer");
    const size_t smem = (size_t)KH * KW * 3 * Cout * 4;
    cudaError_t e = cudaFuncSetAttribute(thin_dgrad3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    if (e != cudaSuccess) return set_error((int)e, "thin_dgrad3 attr: %s", cudaGetErrorString(e));
    thin_dgrad3_kernel<<<ew_grid_b((long long)N * H * W), 256, smem, ST(stream)>>>(dz, wt, dimg_nchw, N, H, W, CinP, OH, OW, Cout, KH, KW,
                                                                                 stride, pad, c_lo);
    return check_launch("mg_thin_dgrad3");
}
extern "C" int mg_conv_img_bwd(const float* dy_nchw, const float* y_nchw, const float* x, const float* w, float* dz4_ws, float* dx,
                               float* dw, float* db, int N, int H, int W, int Cin, int Cout, int act_in, int act_out, void* stream) {
    if (!dy_nchw || !y_nchw || !x || !w || !dz4_ws || !dx || !dw) return set_error(-1, "mg_conv_img_bwd: null pointer");
    // Cin <= 128: conv_img_wgrad_kernel gives each thread kSlots = 5 of the 9 taps (enough while 256 / Cin >= 2), and its
    // shared-memory tile (340 * (Cin + 1) + 1024 floats) must fit the 200 KB it requests
    if (Cin % 4 != 0 || Cin > 128 || Cout > 3 || 256 % Cin != 0)
        return set_error(-2, "mg_conv_img_bwd: Cin must divide 256 and be <= 128, Cout <= 3");
    cudaError_t e = cudaFuncSetAttribute(conv_img_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_img_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return set_error((int)e, "conv_img_bwd attr: %s", cudaGetErrorString(e));
    conv_img_dz_kernel<<<ew_grid_b((long long)N * H * W), 256, 0, ST(stream)>>>(dy_nchw, y_nchw, dz4_ws, N, Cout, (long long)H * W, act_out);
    count_launch();
    conv_img_dgrad_kernel<<<ew_grid_b((long long)N * H * W * (Cin / 4)), 256, (size_t)9 * 4 * Cin * 4, ST(stream)>>>(dz4_ws, x, w, dx, N, H, W,
                                                                                                                   Cin, Cout, act_in);
    count_launch();
    const int tiles_w = cdivb(W, 32), tiles_h = cdivb(H, 8), num_tiles = tiles_w * tiles_h * N;
    int grid = num_sms() * 2;
    if (grid > num_tiles) grid = num_tiles;
    const size_t smem = ((size_t)340 * (Cin + 1) + 256 * 4) * 4;
    // per-CTA partial sums -> fp64 (order-independent) -> added onto dw / db
    const size_t n_dw = (size_t)Cout * Cin * 9, n_db = db ? (size_t)Cout : 0;
    double* acc = nullptr;
    int rc = acc64_alloc(&acc, n_dw + n_db, ST(stream));
    if (rc) return rc;
    conv_img_wgrad_kernel<<<grid, 256, smem, ST(stream)>>>(dz4_ws, x, acc, db ? acc + n_dw : nullptr, N, H, W, Cin, Cout, act_in,
                                                           tiles_w, tiles_h, num_tiles);
    rc = check_launch("mg_conv_img_bwd");
    if (!rc) rc = acc64_fold(acc, dw, n_dw, 1, ST(stream));
    if (!rc && db) rc = acc64_fold(acc + n_dw, db, n_db, 1, ST(stream));
    const int rc2 = acc64_free(acc, ST(stream));
    return rc ? rc : rc2;
}
extern "C" int mg_conv_to1_bwd(const float* dl, const float* x, const float* w, float* dx, float* dw, float* db, int N, int H, int W,
                               int Cin, int KH, int KW, int pad, int accumulate_dx, void* stream) {
    if (!dl || !x || !w) return set_error(-1, "mg_conv_to1_bwd: null pointer");
    const int OH = H + 2 * pad - KH + 1, OW = W + 2 * pad - KW + 1;
    if (dx) {
        conv_to1_dgrad_kernel<<<ew_grid_b((long long)N * H * W * (Cin / 4)), 256, (size_t)KH * KW * Cin * 4, ST(stream)>>>(dl, w, dx, N, H, W, Cin, KH, KW, pad, OH, OW,
                                                                                                 accumulate_dx);
        count_launch();
    }
    if (dw) {
        // per-block partial sums -> fp64 (order-independent) -> added onto dw / db
        const size_t n_dw = (size_t)Cin * KH * KW, n_db = db ? 1 : 0;
        double* acc = nullptr;
        int rc = acc64_alloc(&acc, n_dw + n_db, ST(stream));
        if (rc) return rc;
        dim3 grid(num_sms() * 4, KH * KW);      // latency-bound per-thread pixel loops: 4x the blocks
        conv_to1_wgrad_kernel<<<grid, 128, 0, ST(stream)>>>(dl, x, acc, db ? acc + n_dw : nullptr, N, H, W, Cin, KH, KW, pad, OH, OW);
        rc = check_launch("mg_conv_to1_bwd");
        if (!rc) rc = acc64_fold(acc, dw, n_dw, 1, ST(stream));
        if (!rc && db) rc = acc64_fold(acc + n_dw, db, n_db, 1, ST(stream));
        const int rc2 = acc64_free(acc, ST(stream));
        return rc ? rc : rc2;
    }
    return check_launch("mg_conv_to1_bwd");
}
extern "C" int mg_avgpool3s2_bwd(const float* dout, float* din, int N, int H, int W, int C, int OH, int OW, void* stream) {
    if (!dout || !din) return set_error(-1, "mg_avgpool3s2_bwd: null pointer");
    avgpool3s2_bwd_kernel<<<ew_grid_b((long long)N * H * W * (C / 4)), 256, 0, ST(stream)>>>(dout, din, N, H, W, C, OH, OW);
    return check_launch("mg_avgpool3s2_bwd");
}
extern "C" int mg_reflect_pad_bwd(const float* dpad, float* dx, int N, int H, int W, int C, int pad, int accumulate, void* stream) {
    if (!dpad || !dx) return set_error(-1, "mg_reflect_pad_bwd: null pointer");
    reflect_pad_bwd_kernel<<<ew_grid_b((long long)N * H * W * (C / 4)), 256, 0, ST(stream)>>>(dpad, dx, N, H, W, C, pad, accumulate);
    return check_launch("mg_reflect_pad_bwd");
}
extern "C" int mg_resize_bilinear_bwd(const float* dout, float* din_zeroed, int N, int H, int W, int C, int OH, int OW, void* stream) {
    if (!dout || !din_zeroed) return set_error(-1, "mg_resize_bilinear_bwd: null pointer");
    const size_t n = (size_t)N * H * W * C;
    double* acc = nullptr;
    int rc = acc64_alloc(&acc, n, ST(stream));
    if (rc) return rc;
    resize_bilinear_bwd_kernel<<<ew_grid_b((long long)N * OH * OW * C), 256, 0, ST(stream)>>>(dout, acc, N, H, W, C, OH, OW);
    rc = check_launch("mg_resize_bilinear_bwd");
    if (!rc) rc = acc64_fold(acc, din_zeroed, n, 1, ST(stream));
    const int rc2 = acc64_free(acc, ST(stream));
    return rc ? rc : rc2;
}
extern "C" int mg_masked_mean_bcast_bwd(const float* dout, const float* mref, const float* mtag, float* dx, int N, int h, int w, int C,
                                        int MH, int MW, void* stream) {
    if (!dout || !mref || !mtag || !dx) return set_error(-1, "mg_masked_mean_bcast_bwd: null pointer");
    dim3 grid(cdivb(C, 32), N);
    masked_mean_bcast_bwd_kernel<<<grid, 256, 0, ST(stream)>>>(dout, mref, mtag, dx, N, h, w, C, MH, MW);
    return check_launch("mg_masked_mean_bcast_bwd");
}
extern "C" int mg_spectral_norm_bwd(const float* dwt, const float* w_orig, const float* u, const float* v, const float* inv_sigma,
                                    double* dot_ws, float* dw, int O, long long K, int accumulate, void* stream) {
    if (!dwt || !w_orig || !u || !v || !inv_sigma || !dot_ws || !dw) return set_error(-1, "mg_spectral_norm_bwd: null pointer");
    cudaMemsetAsync(dot_ws, 0, sizeof(double), ST(stream));
    sn_bwd_dot_kernel<<<ew_grid_b((long long)O * K), 256, 0, ST(stream)>>>(dwt, w_orig, (long long)O * K, dot_ws);
    count_launch();
    sn_bwd_apply_kernel<<<ew_grid_b((long long)O * K), 256, 0, ST(stream)>>>(dwt, u, v, inv_sigma, dot_ws, dw, O, K, accumulate);
    return check_launch("mg_spectral_norm_bwd");
}
extern "C" int mg_pack_weight_dgrad_gb(const float* wg, const float* wb, float* out, int C, int I, int BN, void* stream) {
    if (!wg || !wb || !out) return set_error(-1, "mg_pack_weight_dgrad_gb: null pointer");
    pack_weight_dgrad_gb_kernel<<<ew_grid_b((long long)I * 9 * 2 * C), 256, 0, ST(stream)>>>(wg, wb, out, C, I, BN);
    return check_launch("mg_pack_weight_dgrad_gb");
}
extern "C" int mg_unpack_wgrad_gb(const float* dwp, float* dwg, float* dwb, int C, int I, int BN, int accumulate, void* stream) {
    if (!dwp || !dwg || !dwb) return set_error(-1, "mg_unpack_wgrad_gb: null pointer");
    unpack_wgrad_gb_kernel<<<ew_grid_b(2LL * C * I * 9), 256, 0, ST(stream)>>>(dwp, dwg, dwb, C, I, BN, accumulate);
    return check_launch("mg_unpack_wgrad_gb");
}
