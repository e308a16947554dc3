// michigan_b200 — VGG19 perceptual loss and Lab colour loss (sm_90a; reference models/networks/loss.py:178-207 VGGLoss,
// 403-531 LabColorLoss, architecture.py:160-190 VGG19).
//
// The VGG19 convolutions run on the existing kernels (conv_thin for conv1_1, the wgmma implicit-GEMM / 3x3 group kernels for
// the rest, conv_dgrad / thin_dgrad3 backward) and the five L1 terms on mg_loss_reduce.  What the network adds is here:
//   mg_maxpool2_nhwc      2x2 / stride 2 max-pool (floor mode) of an fp32 or 16-bit NHWC tensor, writing fp32 and/or the 16-bit
//                         operand of the next conv;
//   mg_maxpool2_relu_bwd  its gather-form backward fused with the preceding ReLU's: the arg-max is recomputed from the same saved
//                         tensor the forward pooled, so both agree bit for bit; fp32 and/or bf16 (conv_dgrad's dy16) out;
//   mg_relu_bwd16         ReLU backward of the layers without a pool, same outputs;
//   mg_lab_loss_fwd/bwd   the Lab colour L1 loss over fake and real in one pass; d fake written directly (NCHW);
//   mg_hair_avg_lab_fwd/bwd  HairAvgLabLoss (loss.py:534-621): masked per-image Lab sums of fake and real, and d fake;
//   mg_style_loss_fwd     the style loss of StyleContentLoss (loss.py:624-711) for every tap in one launch, from mg_in_stats' sums;
//   mg_style_tap_grad     its gradient w.r.t. one fake tap, with the content loss's folded in at relu5_1, added to the VGG L1's;
//   mg_pixel_l1_fwd/bwd   the background (masked) and rgb L1 losses on the images (loss.py:388-400, pix2pix_model.py:328-333).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "mg_internal.h"
#include "mg_lab.cuh"

namespace mg {

// ------------------------------------------------------------------------------------------------ 8-channel vectors
// Every thread of the pooling / ReLU kernels owns 8 consecutive channels: one 16-byte load of a 16-bit tensor, two of fp32.
__device__ __forceinline__ void load8(const float* a32, const uint16_t* a16, int fmt, size_t off, float v[8]) {
    if (a32) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(a32 + off));
        const float4 y = __ldg(reinterpret_cast<const float4*>(a32 + off + 4));
        v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; v[4] = y.x; v[5] = y.y; v[6] = y.z; v[7] = y.w;
    } else {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(a16 + off));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint16_t lo = (uint16_t)(w[i] & 0xffffu), hi = (uint16_t)(w[i] >> 16);
            if (fmt == 1) {
                v[2 * i] = __half2float(__ushort_as_half(lo)); v[2 * i + 1] = __half2float(__ushort_as_half(hi));
            } else {
                v[2 * i] = __bfloat162float(__ushort_as_bfloat16(lo)); v[2 * i + 1] = __bfloat162float(__ushort_as_bfloat16(hi));
            }
        }
    }
}

__device__ __forceinline__ void store8_32(float* p, size_t off, const float v[8]) {
    *reinterpret_cast<float4*>(p + off) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + off + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// round to nearest; fp16 clamped to its finite range (the out16 convention of the conv epilogues)
__device__ __forceinline__ uint16_t to16(float v, int fmt) {
    if (fmt == 1) return __half_as_ushort(__float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f)));
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}

__device__ __forceinline__ void store8_16(uint16_t* p, size_t off, const float v[8], int fmt) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) w[i] = (uint32_t)to16(v[2 * i], fmt) | ((uint32_t)to16(v[2 * i + 1], fmt) << 16);
    *reinterpret_cast<uint4*>(p + off) = make_uint4(w[0], w[1], w[2], w[3]);
}

// torch's max_pool2d rule: a later element replaces the running maximum if it is larger or NaN, so ties keep the first
// element in row-major window order
__device__ __forceinline__ bool pool_takes(float v, float m) { return v > m || isnan(v); }

// ------------------------------------------------------------------------------------------------ max-pool forward
__global__ void __launch_bounds__(256) maxpool2_kernel(const float* __restrict__ in32, const uint16_t* __restrict__ in16, int in_fmt,
                                                       float* __restrict__ out32, uint16_t* __restrict__ out16, int out_fmt, int N,
                                                       int H, int W, int C, int OH, int OW) {
    const int cg = C / 8;
    const long long total = (long long)N * OH * OW * cg;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % cg) * 8;
        long long r = idx / cg;
        const int ow = (int)(r % OW); r /= OW;
        const int oh = (int)(r % OH);
        const int n = (int)(r / OH);
        const size_t p00 = (((size_t)n * H + 2 * oh) * W + 2 * ow) * C + c;
        const size_t offs[4] = {p00, p00 + C, p00 + (size_t)W * C, p00 + (size_t)W * C + C};
        float m[8], v[8];
        load8(in32, in16, in_fmt, offs[0], m);
#pragma unroll
        for (int k = 1; k < 4; ++k) {
            load8(in32, in16, in_fmt, offs[k], v);
#pragma unroll
            for (int i = 0; i < 8; ++i) m[i] = pool_takes(v[i], m[i]) ? v[i] : m[i];
        }
        const size_t o = (size_t)idx * 8;
        if (out32) store8_32(out32, o, m);
        if (out16) store8_16(out16, o, m, out_fmt);
    }
}

// ------------------------------------------------------------------------------------------------ max-pool + ReLU backward
// One thread per (2x2 window, 8 channels), windows covering the whole input (ceil): the last row / column of an odd-sized
// input belongs to no pooled window and receives only `add`.  g = (window arg-max ? dpool : 0) + add;  dx = [a > 0] * g.
__global__ void __launch_bounds__(256) maxpool2_relu_bwd_kernel(const float* __restrict__ dpool, const float* __restrict__ a32,
                                                                const uint16_t* __restrict__ a16, int a_fmt, const float* add,
                                                                float* dx32, __nv_bfloat16* __restrict__ dx16, int N, int H, int W,
                                                                int C) {
    const int OH = H / 2, OW = W / 2, WH = (H + 1) / 2, WW = (W + 1) / 2;
    const int cg = C / 8;
    const long long total = (long long)N * WH * WW * cg;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % cg) * 8;
        long long r = idx / cg;
        const int ww = (int)(r % WW); r /= WW;
        const int wh = (int)(r % WH);
        const int n = (int)(r / WH);
        const bool pooled = wh < OH && ww < OW;
        float a[4][8];
        bool have[4];
        size_t offs[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int y = 2 * wh + (k >> 1), x = 2 * ww + (k & 1);
            have[k] = y < H && x < W;
            offs[k] = (((size_t)n * H + y) * W + x) * C + c;
            if (have[k]) load8(a32, a16, a_fmt, offs[k], a[k]);
        }
        float dp[8];
        int arg[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { dp[i] = 0.f; arg[i] = -1; }
        if (pooled) {
            load8(dpool, nullptr, 0, (((size_t)n * OH + wh) * OW + ww) * C + c, dp);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float m = a[0][i];
                int best = 0;
#pragma unroll
                for (int k = 1; k < 4; ++k)
                    if (pool_takes(a[k][i], m)) { m = a[k][i]; best = k; }
                arg[i] = best;
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (!have[k]) continue;
            float g[8], ad[8];
            if (add) load8(add, nullptr, 0, offs[k], ad);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float t = arg[i] == k ? dp[i] : 0.f;
                if (add) t += ad[i];
                g[i] = a[k][i] > 0.f ? t : 0.f;
            }
            if (dx32) store8_32(dx32, offs[k], g);
            if (dx16) store8_16(reinterpret_cast<uint16_t*>(dx16), offs[k], g, 2);
        }
    }
}

// ------------------------------------------------------------------------------------------------ ReLU backward
// dz = [a > 0] * (dy + add), over n elements (n % 8 == 0).
__global__ void __launch_bounds__(256) relu_bwd16_kernel(const float* dy, const float* add, const float* __restrict__ a32,
                                                         const uint16_t* __restrict__ a16, int a_fmt, float* dz32,
                                                         __nv_bfloat16* __restrict__ dz16, long long n8) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
        const size_t off = (size_t)i * 8;
        float a[8], d[8], ad[8], g[8];
        load8(a32, a16, a_fmt, off, a);
        load8(dy, nullptr, 0, off, d);
        if (add) load8(add, nullptr, 0, off, ad);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float t = add ? d[k] + ad[k] : d[k];
            g[k] = a[k] > 0.f ? t : 0.f;
        }
        if (dz32) store8_32(dz32, off, g);
        if (dz16) store8_16(reinterpret_cast<uint16_t*>(dz16), off, g, 2);
    }
}

// ------------------------------------------------------------------------------------------------ Lab colour loss
// loss.py:403-531 (balance_Lab = False), per pixel as mg_lab.cuh.  L (channel 0) never enters the loss; the balanced loss is
// mg_loss_reduce op 11 (mg_loss.cu).
// sums[0] += sum over pixels of |a_fake - a_real| + |b_fake - b_real|  (fp64, caller zeroes)
__global__ void __launch_bounds__(256) lab_loss_fwd_kernel(const float* __restrict__ fake, const float* __restrict__ real,
                                                           double* __restrict__ sums, int N, long long HW) {
    double s = 0.0;
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long n = idx / HW, p = idx - n * HW;
        float tf[3], tr[3], ff[3], fr[3];
        lab_xyz(fake + (size_t)n * 3 * HW, (size_t)HW, (size_t)p, tf);
        lab_xyz(real + (size_t)n * 3 * HW, (size_t)HW, (size_t)p, tr);
#pragma unroll
        for (int k = 0; k < 3; ++k) { ff[k] = lab_f(tf[k]); fr[k] = lab_f(tr[k]); }
        const float da = 500.f * (ff[0] - ff[1]) - 500.f * (fr[0] - fr[1]);
        const float db = 200.f * (ff[1] - ff[2]) - 200.f * (fr[1] - fr[2]);
        s += (double)fabsf(da) + (double)fabsf(db);
    }
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    __shared__ double part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += part[i];
        atomicAdd(sums, t);
    }
}

// dfake = gscale[0] * d(sum |da| + |db|) / d fake
__global__ void __launch_bounds__(256) lab_loss_bwd_kernel(const float* __restrict__ fake, const float* __restrict__ real,
                                                           const float* __restrict__ gscale, float* __restrict__ dfake, int N,
                                                           long long HW) {
    const float g = __ldg(gscale);
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long n = idx / HW, p = idx - n * HW;
        float tf[3], tr[3], ff[3], fr[3];
        lab_xyz(fake + (size_t)n * 3 * HW, (size_t)HW, (size_t)p, tf);
        lab_xyz(real + (size_t)n * 3 * HW, (size_t)HW, (size_t)p, tr);
#pragma unroll
        for (int k = 0; k < 3; ++k) { ff[k] = lab_f(tf[k]); fr[k] = lab_f(tr[k]); }
        const float sa = sgn(500.f * (ff[0] - ff[1]) - 500.f * (fr[0] - fr[1]));
        const float sb = sgn(200.f * (ff[1] - ff[2]) - 200.f * (fr[1] - fr[2]));
        lab_ab_backprop(tf, ff, sa, sb, g, dfake + (size_t)n * 3 * HW + p, (size_t)HW);
    }
}

// ------------------------------------------------------------------------------------------------ hair-average Lab loss
// HairAvgLabLoss (loss.py:571-577, 601-621): avg = sum(Lab * m) / sum(m) per image (a mask sum of 0 counts as 1), L1 over the
// a, b averages of fake and real.  Grid (blocks per image, N); every block reduces its share of one image in a fixed order and
// writes its 8 partial sums, then hair_avg_lab_sum_kernel adds the partials of each image in a fixed order: no atomics, so two
// runs give the same bits.  Per image: [fake: m L, m a, m b, m | real: the same] (each product rounded to fp32 first, as
// torch's `input * mask`).
constexpr int kHairVals = 8;

__global__ void __launch_bounds__(256) hair_avg_lab_part_kernel(const float* __restrict__ fake, const float* __restrict__ real,
                                                                const float* __restrict__ mfake, const float* __restrict__ mreal,
                                                                double* __restrict__ part, long long HW) {
    const int n = blockIdx.y;
    double s[kHairVals];
#pragma unroll
    for (int k = 0; k < kHairVals; ++k) s[k] = 0.0;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float m = __ldg((i ? mreal : mfake) + (size_t)n * HW + p);
            if (m == 0.f) continue;
            float t[3], f[3];
            lab_xyz((i ? real : fake) + (size_t)n * 3 * HW, (size_t)HW, (size_t)p, t);
#pragma unroll
            for (int k = 0; k < 3; ++k) f[k] = lab_f(t[k]);
            // loss.py:563-569: L = 116 f(Y) - 16 above the threshold, 903.3 Y below
            const float L = t[1] > kLabT ? 116.f * f[1] - 16.f : 903.3f * t[1];
            s[4 * i + 0] += (double)__fmul_rn(L, m);
            s[4 * i + 1] += (double)__fmul_rn(500.f * (f[0] - f[1]), m);
            s[4 * i + 2] += (double)__fmul_rn(200.f * (f[1] - f[2]), m);
            s[4 * i + 3] += (double)m;
        }
    }
    __shared__ double red[8][kHairVals];
#pragma unroll
    for (int k = 0; k < kHairVals; ++k) {
        for (int off = 16; off > 0; off >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], off);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = s[k];
    }
    __syncthreads();
    if (threadIdx.x < kHairVals) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
        part[((size_t)n * gridDim.x + blockIdx.x) * kHairVals + threadIdx.x] = t;
    }
}

// One block per image, one warp per value: sums[n][k] = sum over the image's nb partials, in a fixed order.
__global__ void __launch_bounds__(256) hair_avg_lab_sum_kernel(const double* __restrict__ part, double* __restrict__ sums, int nb) {
    const int n = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const double* p = part + (size_t)n * nb * kHairVals + k;
    double s = 0.0;
    for (int b = lane; b < nb; b += 32) s += p[(size_t)b * kHairVals];
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) sums[(size_t)n * kHairVals + k] = s;
}

// dfake = mask_fake * (T[n][0] da/dimg + T[n][1] db/dimg), T[n][j] = g / (2N) sgn(avg_f - avg_r) / cnt_f, formed per block
// from the image's sums (loss.py:575 replaces a zero mask sum by 1).
__global__ void __launch_bounds__(256) hair_avg_lab_bwd_kernel(const float* __restrict__ fake, const float* __restrict__ mfake,
                                                               const double* __restrict__ sums, const float* __restrict__ gscale,
                                                               float* __restrict__ dfake, long long HW) {
    const int n = blockIdx.y;
    __shared__ float tab[2];
    if (threadIdx.x < 2) {
        const double* s = sums + (size_t)n * kHairVals;
        const double cf = s[3] == 0.0 ? 1.0 : s[3], cr = s[7] == 0.0 ? 1.0 : s[7];
        const double d = s[1 + threadIdx.x] / cf - s[5 + threadIdx.x] / cr;
        const double sg = d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0);
        tab[threadIdx.x] = (float)((double)__ldg(gscale) / (2.0 * gridDim.y) * sg / cf);
    }
    __syncthreads();
    const float ta = tab[0], tb = tab[1];
    const float* img = fake + (size_t)n * 3 * HW;
    float* out = dfake + (size_t)n * 3 * HW;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
        const float m = __ldg(mfake + (size_t)n * HW + p);
        if (m == 0.f) {
#pragma unroll
            for (int c = 0; c < 3; ++c) out[c * HW + p] = 0.f;
            continue;
        }
        float t[3], f[3];
        lab_xyz(img, (size_t)HW, (size_t)p, t);
#pragma unroll
        for (int k = 0; k < 3; ++k) f[k] = lab_f(t[k]);
        lab_ab_backprop(t, f, ta, tb, m, out + p, (size_t)HW);
    }
}

// ------------------------------------------------------------------------------------------------ style loss
// calc_mean_std (loss.py:624-632) from the fp64 per-(n, c) sums of mg_in_stats ([N][2][C]: sum x, then sum x^2, over M pixels):
//   mu = S1 / M,  var = (S2 - S1 mu) / (M - 1) (unbiased; clamped at 0 against cancellation),  sigma = sqrt(var + 1e-5).
// calc_style_loss (loss.py:668-683, remove_background False) of one tap: MSE(mu_f, mu_t) + MSE(sigma_f, sigma_t) over N x C.
//
// Masked mode (cnt_f, cnt_t set; calc_mean_std_mask, loss.py:634-654, and calc_style_loss with remove_background, 679-694): the
// sums are mg_loss_reduce op 10's (sum m x, sum m x^2 per (n, c)) and cnt the per-image sum m, m binary (m^2 = m), D = cnt:
//   mu = S1 / (D + eps),  var = sum m (x - mu)^2 / (D + eps) + eps = (S2 - mu (2 S1 - mu D)) / (D + eps) + eps  (biased, eps
//   twice, no M - 1: no pixel-count refusal; an image without mask pixels gives mu = 0, sigma = sqrt(eps)).
// coef then holds op 10's backward table: mu' = mu (1 + eps / (D + eps)), A = 2 (mu_f - mu_t) / (N C (D + eps)),
// B = 2 (sigma_f - sigma_t) / (N C sigma_f (D + eps)).  mu' folds in the term -(m_p / (D + eps)) sum_q m_q (x_q - mu) =
// -m_p mu eps / (D + eps) of d var / d x_p, which is not zero because of the eps in mu's denominator.
struct StyleTap {
    const double* sums_f;   // [N][2][C] of the fake images
    const double* sums_t;   // [N][2][C] of the style targets
    float* coef;            // [N][3][C] out: mu_f, mu_f - mu_t, (sigma_f - sigma_t) / sigma_f  (masked: mu', A, B)
    long long M;
    int N, C;
    // appended: the masked mode (both null: unmasked)
    const double* cnt_f;    // [N] sum m of the fake images' masks
    const double* cnt_t;    // [N] sum m of the style targets' masks
};
constexpr int kMaxStyleTaps = 8;
struct StyleTaps {
    StyleTap t[kMaxStyleTaps];
    int n;
};
constexpr double kStyleEps = 1e-5;

// One block for every tap (N*C is at most a few thousand per tap): the per-tap sums are added in a fixed order, so the loss is
// bit-reproducible.  loss[0] += sum over taps of (sum (mu_f - mu_t)^2 + (sigma_f - sigma_t)^2) / (N*C).
__global__ void __launch_bounds__(512) style_loss_fwd_kernel(const StyleTaps taps, double* __restrict__ loss) {
    __shared__ double part[16];
    double total = 0.0;
    for (int k = 0; k < taps.n; ++k) {
        const StyleTap t = taps.t[k];
        const int NC = t.N * t.C;
        const double M = (double)t.M;
        double s = 0.0;
        for (int i = threadIdx.x; i < NC; i += blockDim.x) {
            const int n = i / t.C, c = i - n * t.C;
            const double* f = t.sums_f + (size_t)n * 2 * t.C;
            const double* r = t.sums_t + (size_t)n * 2 * t.C;
            float* co = t.coef + (size_t)n * 3 * t.C + c;
            if (t.cnt_f) {
                const double Df = t.cnt_f[n], Dt = t.cnt_t[n], ef = Df + kStyleEps, et = Dt + kStyleEps;
                const double mf = f[c] / ef, mt = r[c] / et;
                const double sf = sqrt(fmax(f[t.C + c] - mf * (2.0 * f[c] - mf * Df), 0.0) / ef + kStyleEps);
                const double st = sqrt(fmax(r[t.C + c] - mt * (2.0 * r[c] - mt * Dt), 0.0) / et + kStyleEps);
                const double dm = mf - mt, ds = sf - st;
                s += dm * dm + ds * ds;
                co[0] = (float)(mf * (1.0 + kStyleEps / ef));
                co[t.C] = (float)(2.0 * dm / ((double)NC * ef));
                co[2 * t.C] = (float)(2.0 * ds / ((double)NC * sf * ef));
                continue;
            }
            const double mf = f[c] / M, mt = r[c] / M;
            const double sf = sqrt(fmax((f[t.C + c] - f[c] * mf) / (M - 1.0), 0.0) + kStyleEps);
            const double st = sqrt(fmax((r[t.C + c] - r[c] * mt) / (M - 1.0), 0.0) + kStyleEps);
            const double dm = mf - mt, ds = sf - st;
            s += dm * dm + ds * ds;
            co[0] = (float)mf;
            co[t.C] = (float)dm;
            co[2 * t.C] = (float)(ds / sf);
        }
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            double b = 0.0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b += part[w];
            total += b / (double)NC;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) loss[0] += total;
}

// Gradient w.r.t. one fake tap [N, HW, C] (4 channels per thread, 128-bit loads and stores):
//   out = add + g_s [ka (mu_f - mu_t) + kb (sigma_f - sigma_t) / sigma_f (x - mu_f)] + g_c kc (x - t)
// ka = 2 / (N C M), kb = 2 / (N C (M - 1)), kc = 2 / numel; the style part is skipped without coef, the content part without t.
// add may alias out (each element is read before it is written by the same thread).
__global__ void __launch_bounds__(256) style_tap_grad_kernel(const float* __restrict__ x, const float* __restrict__ coef,
                                                             const float* __restrict__ tgt, const float* add, float* out,
                                                             const float* __restrict__ g, long long HW, int C, float ka, float kb,
                                                             float kc, long long total4) {
    const float gs = coef ? __ldg(g) : 0.f, gc = tgt ? __ldg(g + 1) : 0.f;
    const int c4 = C / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4) * 4;
        const long long n = i / (HW * c4);
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
        float r[4] = {0.f, 0.f, 0.f, 0.f};
        if (add) {
            const float4 a = reinterpret_cast<const float4*>(add)[i];
            r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w;
        }
        if (coef) {
            const float* co = coef + (size_t)n * 3 * C + c;
            const float4 mu = __ldg(reinterpret_cast<const float4*>(co));
            const float4 dm = __ldg(reinterpret_cast<const float4*>(co + C));
            const float4 ds = __ldg(reinterpret_cast<const float4*>(co + 2 * C));
            const float m[4] = {mu.x, mu.y, mu.z, mu.w}, a[4] = {dm.x, dm.y, dm.z, dm.w}, b[4] = {ds.x, ds.y, ds.z, ds.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) r[j] += gs * (ka * a[j] + kb * b[j] * (xs[j] - m[j]));
        }
        if (tgt) {
            const float4 tv = __ldg(reinterpret_cast<const float4*>(tgt) + i);
            const float ts[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) r[j] += gc * (kc * (xs[j] - ts[j]));
        }
        reinterpret_cast<float4*>(out)[i] = make_float4(r[0], r[1], r[2], r[3]);
    }
}

// ------------------------------------------------------------------------------------------------ pixel L1 (background / rgb)
// RGBBackgroundL1Loss (loss.py:388-400): L1(fake * m, tag * m), m = input_semantics[:, 0] broadcast over the 3 channels; the rgb
// loss (pix2pix_model.py:51, 328-333) is the same without m.  Both products are rounded before the difference, as torch does.
__device__ __forceinline__ float pixel_diff(float f, float t, const float* m, size_t mi) {
    if (!m) return f - t;
    const float mv = __ldg(m + mi);
    return __fmul_rn(f, mv) - __fmul_rn(t, mv);
}

__global__ void __launch_bounds__(256) pixel_l1_fwd_kernel(const float* __restrict__ fake, const float* __restrict__ tag,
                                                           const float* __restrict__ mask, double* __restrict__ sums, int N,
                                                           long long HW) {
    double s = 0.0;
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long n = idx / HW, p = idx - n * HW;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t o = ((size_t)n * 3 + c) * HW + p;
            s += (double)fabsf(pixel_diff(__ldg(fake + o), __ldg(tag + o), mask, (size_t)idx));
        }
    }
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    __shared__ double part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += part[i];
        atomicAdd(sums, t);
    }
}

// dfake = (gscale[0] * sign(m f - m t)) * m, sign(0) = 0
__global__ void __launch_bounds__(256) pixel_l1_bwd_kernel(const float* __restrict__ fake, const float* __restrict__ tag,
                                                           const float* __restrict__ mask, const float* __restrict__ gscale,
                                                           float* __restrict__ dfake, int N, long long HW) {
    const float g = __ldg(gscale);
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long n = idx / HW, p = idx - n * HW;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t o = ((size_t)n * 3 + c) * HW + p;
            const float d = g * sgn(pixel_diff(__ldg(fake + o), __ldg(tag + o), mask, (size_t)idx));
            dfake[o] = mask ? d * __ldg(mask + idx) : d;
        }
    }
}

static int grid_for(long long work) {
    long long g = (work + 255) / 256;
    const long long cap = (long long)num_sms() * 16;
    if (g > cap) g = cap;
    return (int)(g < 1 ? 1 : g);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace mg

using namespace mg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mg_maxpool2_nhwc(const float* in32, const void* in16, int in_fmt, float* out32, void* out16, int out_fmt, int N, int H,
                                int W, int C, void* stream) {
    if ((!in32) == (!in16)) return set_error(-1, "mg_maxpool2_nhwc: exactly one of in32 / in16 must be given");
    if (!out32 && !out16) return set_error(-1, "mg_maxpool2_nhwc: null output");
    if ((in16 && (in_fmt < 1 || in_fmt > 2)) || (out16 && (out_fmt < 1 || out_fmt > 2)))
        return set_error(-3, "mg_maxpool2_nhwc: 16-bit formats are 1 (fp16) or 2 (bf16)");
    if (N < 1 || H < 2 || W < 2 || C < 8 || C % 8 != 0) return set_error(-2, "mg_maxpool2_nhwc: bad size (C must be a multiple of 8)");
    if (!aligned16(in32 ? (const void*)in32 : in16) || (out32 && !aligned16(out32)) || (out16 && !aligned16(out16)))
        return set_error(-4, "mg_maxpool2_nhwc: tensors must be 16-byte aligned");
    const int OH = H / 2, OW = W / 2;
    maxpool2_kernel<<<grid_for((long long)N * OH * OW * (C / 8)), 256, 0, ST(stream)>>>(
        in32, static_cast<const uint16_t*>(in16), in_fmt, out32, static_cast<uint16_t*>(out16), out_fmt, N, H, W, C, OH, OW);
    return check_launch("mg_maxpool2_nhwc");
}

extern "C" int mg_maxpool2_relu_bwd(const float* dpool, const float* a32, const void* a16, int a_fmt, const float* add, float* dx32,
                                    void* dx16, int N, int H, int W, int C, void* stream) {
    if (!dpool || (!a32) == (!a16)) return set_error(-1, "mg_maxpool2_relu_bwd: need dpool and exactly one of a32 / a16");
    if (!dx32 && !dx16) return set_error(-1, "mg_maxpool2_relu_bwd: null output");
    if (a16 && (a_fmt < 1 || a_fmt > 2)) return set_error(-3, "mg_maxpool2_relu_bwd: 16-bit formats are 1 (fp16) or 2 (bf16)");
    if (N < 1 || H < 2 || W < 2 || C < 8 || C % 8 != 0) return set_error(-2, "mg_maxpool2_relu_bwd: bad size (C must be a multiple of 8)");
    if (!aligned16(dpool) || !aligned16(a32 ? (const void*)a32 : a16) || (add && !aligned16(add)) || (dx32 && !aligned16(dx32)) ||
        (dx16 && !aligned16(dx16)))
        return set_error(-4, "mg_maxpool2_relu_bwd: tensors must be 16-byte aligned");
    maxpool2_relu_bwd_kernel<<<grid_for((long long)N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8)), 256, 0, ST(stream)>>>(
        dpool, a32, static_cast<const uint16_t*>(a16), a_fmt, add, dx32, static_cast<__nv_bfloat16*>(dx16), N, H, W, C);
    return check_launch("mg_maxpool2_relu_bwd");
}

extern "C" int mg_relu_bwd16(const float* dy, const float* add, const float* a32, const void* a16, int a_fmt, float* dz32, void* dz16,
                             long long n, void* stream) {
    if (!dy || (!a32) == (!a16)) return set_error(-1, "mg_relu_bwd16: need dy and exactly one of a32 / a16");
    if (!dz32 && !dz16) return set_error(-1, "mg_relu_bwd16: null output");
    if (a16 && (a_fmt < 1 || a_fmt > 2)) return set_error(-3, "mg_relu_bwd16: 16-bit formats are 1 (fp16) or 2 (bf16)");
    if (n < 8 || n % 8 != 0) return set_error(-2, "mg_relu_bwd16: element count must be a positive multiple of 8");
    if (!aligned16(dy) || !aligned16(a32 ? (const void*)a32 : a16) || (add && !aligned16(add)) || (dz32 && !aligned16(dz32)) ||
        (dz16 && !aligned16(dz16)))
        return set_error(-4, "mg_relu_bwd16: tensors must be 16-byte aligned");
    relu_bwd16_kernel<<<grid_for(n / 8), 256, 0, ST(stream)>>>(dy, add, a32, static_cast<const uint16_t*>(a16), a_fmt, dz32,
                                                              static_cast<__nv_bfloat16*>(dz16), n / 8);
    return check_launch("mg_relu_bwd16");
}

extern "C" int mg_lab_loss_fwd(const float* fake_nchw, const float* real_nchw, double* sums, int N, int H, int W, void* stream) {
    if (!fake_nchw || !real_nchw || !sums) return set_error(-1, "mg_lab_loss_fwd: null pointer");
    if (N < 1 || H < 1 || W < 1) return set_error(-2, "mg_lab_loss_fwd: bad size");
    lab_loss_fwd_kernel<<<grid_for((long long)N * H * W), 256, 0, ST(stream)>>>(fake_nchw, real_nchw, sums, N, (long long)H * W);
    return check_launch("mg_lab_loss_fwd");
}

extern "C" int mg_lab_loss_bwd(const float* fake_nchw, const float* real_nchw, const float* gscale, float* dfake_nchw, int N, int H, int W,
                               void* stream) {
    if (!fake_nchw || !real_nchw || !gscale || !dfake_nchw) return set_error(-1, "mg_lab_loss_bwd: null pointer");
    if (N < 1 || H < 1 || W < 1) return set_error(-2, "mg_lab_loss_bwd: bad size");
    lab_loss_bwd_kernel<<<grid_for((long long)N * H * W), 256, 0, ST(stream)>>>(fake_nchw, real_nchw, gscale, dfake_nchw, N,
                                                                               (long long)H * W);
    return check_launch("mg_lab_loss_bwd");
}

// blocks per image of the hair-average kernels: enough to fill the GPU, no more than the image has 256-pixel chunks
static int hair_blocks(int N, long long HW) {
    long long b = (HW + 255) / 256;
    const long long cap = ((long long)num_sms() * 8 + N - 1) / N;
    if (b > cap) b = cap;
    return (int)(b < 1 ? 1 : b);
}

extern "C" int mg_hair_avg_lab_fwd(const float* fake_nchw, const float* real_nchw, const float* mask_fake, const float* mask_real,
                                   double* sums, int N, int H, int W, void* stream) {
    if (!fake_nchw || !real_nchw || !mask_fake || !mask_real || !sums) return set_error(-1, "mg_hair_avg_lab_fwd: null pointer");
    if (N < 1 || N > 65535 || H < 1 || W < 1) return set_error(-2, "mg_hair_avg_lab_fwd: bad size");
    const long long HW = (long long)H * W;
    const int nb = hair_blocks(N, HW);
    double* part = nullptr;
    int rc = acc64_alloc(&part, (size_t)N * nb * kHairVals, ST(stream));
    if (rc) return rc;
    hair_avg_lab_part_kernel<<<dim3(nb, N), 256, 0, ST(stream)>>>(fake_nchw, real_nchw, mask_fake, mask_real, part, HW);
    rc = check_launch("mg_hair_avg_lab_fwd");
    if (!rc) {
        hair_avg_lab_sum_kernel<<<N, 32 * kHairVals, 0, ST(stream)>>>(part, sums, nb);
        rc = check_launch("mg_hair_avg_lab_fwd");
    }
    const int rc2 = acc64_free(part, ST(stream));
    return rc ? rc : rc2;
}

extern "C" int mg_hair_avg_lab_bwd(const float* fake_nchw, const float* mask_fake, const double* sums, const float* gscale,
                                   float* dfake_nchw, int N, int H, int W, void* stream) {
    if (!fake_nchw || !mask_fake || !sums || !gscale || !dfake_nchw) return set_error(-1, "mg_hair_avg_lab_bwd: null pointer");
    if (N < 1 || N > 65535 || H < 1 || W < 1) return set_error(-2, "mg_hair_avg_lab_bwd: bad size");
    const long long HW = (long long)H * W;
    hair_avg_lab_bwd_kernel<<<dim3(hair_blocks(N, HW), N), 256, 0, ST(stream)>>>(fake_nchw, mask_fake, sums, gscale, dfake_nchw, HW);
    return check_launch("mg_hair_avg_lab_bwd");
}

extern "C" int mg_style_loss_fwd(const void* taps_host, int n_taps, double* loss, void* stream) {
    if (!taps_host || !loss) return set_error(-1, "mg_style_loss_fwd: null pointer");
    if (n_taps < 1 || n_taps > kMaxStyleTaps) return set_error(-2, "mg_style_loss_fwd: bad tap count %d", n_taps);
    StyleTaps taps;
    taps.n = n_taps;
    for (int k = 0; k < n_taps; ++k) {
        const StyleTap& t = static_cast<const StyleTap*>(taps_host)[k];
        if (!t.sums_f || !t.sums_t || !t.coef) return set_error(-1, "mg_style_loss_fwd: null pointer in tap %d", k);
        if (t.N < 1 || t.C < 4 || t.C % 4 != 0) return set_error(-2, "mg_style_loss_fwd: bad size in tap %d", k);
        if ((!t.cnt_f) != (!t.cnt_t)) return set_error(-1, "mg_style_loss_fwd: tap %d has one mask count but not the other", k);
        if (!t.cnt_f && t.M < 2)
            return set_error(-2, "mg_style_loss_fwd: tap %d has %lld pixel(s); the unbiased variance needs at least 2 (crop size >= 32)", k,
                             t.M);
        if (!aligned16(t.coef)) return set_error(-4, "mg_style_loss_fwd: coefficient table of tap %d must be 16-byte aligned", k);
        taps.t[k] = t;
    }
    style_loss_fwd_kernel<<<1, 512, 0, ST(stream)>>>(taps, loss);
    return check_launch("mg_style_loss_fwd");
}

extern "C" int mg_style_tap_grad(const float* x, const float* coef, const float* content_t, const float* add, float* out, const float* g,
                                 int N, long long HW, int C, void* stream) {
    if (!x || !out || !g) return set_error(-1, "mg_style_tap_grad: null pointer");
    if (!coef && !content_t) return set_error(-1, "mg_style_tap_grad: neither a style nor a content term");
    if (N < 1 || C < 4 || C % 4 != 0) return set_error(-2, "mg_style_tap_grad: bad size (C must be a multiple of 4)");
    if (coef && HW < 2) return set_error(-2, "mg_style_tap_grad: the style term needs at least 2 pixels");
    if (!aligned16(x) || !aligned16(out) || (coef && !aligned16(coef)) || (content_t && !aligned16(content_t)) || (add && !aligned16(add)))
        return set_error(-4, "mg_style_tap_grad: tensors must be 16-byte aligned");
    const double nc = (double)N * C;
    const float ka = (float)(2.0 / (nc * (double)HW)), kb = (float)(2.0 / (nc * (double)(HW - 1)));
    const long long total4 = (long long)N * HW * (C / 4);
    style_tap_grad_kernel<<<grid_for(total4), 256, 0, ST(stream)>>>(x, coef, content_t, add, out, g, HW, C, ka, kb, ka, total4);
    return check_launch("mg_style_tap_grad");
}

extern "C" int mg_pixel_l1_fwd(const float* fake_nchw, const float* tag_nchw, const float* mask, double* sums, int N, int H, int W,
                               void* stream) {
    if (!fake_nchw || !tag_nchw || !sums) return set_error(-1, "mg_pixel_l1_fwd: null pointer");
    if (N < 1 || H < 1 || W < 1) return set_error(-2, "mg_pixel_l1_fwd: bad size");
    pixel_l1_fwd_kernel<<<grid_for((long long)N * H * W), 256, 0, ST(stream)>>>(fake_nchw, tag_nchw, mask, sums, N, (long long)H * W);
    return check_launch("mg_pixel_l1_fwd");
}

extern "C" int mg_pixel_l1_bwd(const float* fake_nchw, const float* tag_nchw, const float* mask, const float* gscale, float* dfake_nchw,
                               int N, int H, int W, void* stream) {
    if (!fake_nchw || !tag_nchw || !gscale || !dfake_nchw) return set_error(-1, "mg_pixel_l1_bwd: null pointer");
    if (N < 1 || H < 1 || W < 1) return set_error(-2, "mg_pixel_l1_bwd: bad size");
    pixel_l1_bwd_kernel<<<grid_for((long long)N * H * W), 256, 0, ST(stream)>>>(fake_nchw, tag_nchw, mask, gscale, dfake_nchw, N,
                                                                               (long long)H * W);
    return check_launch("mg_pixel_l1_bwd");
}

extern "C" int mg_style_tap_bytes(void) { return (int)sizeof(mg::StyleTap); }
