// michigan_b200 — CUDA-core kernels around the tensor-core implicit GEMM: weight packing, thin
// (3/4/7-channel) direct convolutions, normalisation statistics, input preparation, pooling.
// These are the HBM-bound pieces of the path: coalesced 128-bit accesses, NHWC, no tensor cores.
#include <cuda_runtime.h>
#include <cstdint>
#include <cmath>
#include <cstdlib>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "mg_internal.h"

namespace mg {

__device__ __forceinline__ float rtf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ float act_fn(float v, int act) {
    if (act == MG_ACT_RELU) return fmaxf(v, 0.f);
    if (act == MG_ACT_LRELU) return v > 0.f ? v : 0.2f * v;
    if (act == MG_ACT_TANH) return tanhf(v);
    return v;
}
// 16-bit split: hi = cvt(v), lo = cvt(v - float(hi)); fmt 1 = fp16 (clamped to the finite range), 2 = bf16
__device__ __forceinline__ void split16(float v, int fmt, uint16_t& hi, uint16_t& lo) {
    if (fmt == 1) {
        const __half h = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
        hi = __half_as_ushort(h);
        lo = __half_as_ushort(__float2half_rn(v - __half2float(h)));
    } else {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi = __bfloat16_as_ushort(h);
        lo = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(h)));
    }
}
static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------ weight packing
__global__ void pack_weight_kernel(const float* __restrict__ w, float* __restrict__ out, int O, int I, int KH, int KW,
                                   const float* __restrict__ inv_sigma, int round_) {
    const long long total = (long long)O * KH * KW * I;
    const float s = inv_sigma ? *inv_sigma : 1.f;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = idx % I;
        long long t = idx / I;
        const int kw = t % KW; t /= KW;
        const int kh = t % KH;
        const int o = t / KH;
        float v = w[(((long long)o * I + i) * KH + kh) * KW + kw] * s;
        out[idx] = round_ ? rtf32(v) : v;
    }
}

__global__ void pack_weight_gb_kernel(const float* __restrict__ wg, const float* __restrict__ wb,
                                      float* __restrict__ out, int C, int I, int KH, int KW, int BN) {
    const long long total = 2LL * C * KH * KW * I;
    const int half = BN / 2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = idx % I;
        long long t = idx / I;
        const int kw = t % KW; t /= KW;
        const int kh = t % KH;
        const int R = t / KH;
        const int tile = R / BN, rr = R % BN;
        const float* src = rr < half ? wg : wb;
        const int c = tile * half + (rr < half ? rr : rr - half);
        out[idx] = rtf32(src[(((long long)c * I + i) * KH + kh) * KW + kw]);
    }
}

// 16-bit operands: out[o][tap][part][i], part = hi (and lo when split) of w*inv_sigma
__global__ void pack_weight16_kernel(const float* __restrict__ w, uint16_t* __restrict__ out, int O, int I, int KH, int KW,
                                     const float* __restrict__ inv_sigma, int fmt, int split) {
    const long long total = (long long)O * KH * KW * I;
    const float s = inv_sigma ? *inv_sigma : 1.f;
    const int parts = split ? 2 : 1;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = idx % I;
        long long t = idx / I;
        const int kw = t % KW; t /= KW;
        const int kh = t % KH;
        const int o = t / KH;
        const float v = w[(((long long)o * I + i) * KH + kh) * KW + kw] * s;
        uint16_t hi, lo;
        split16(v, fmt, hi, lo);
        const size_t base = ((size_t)o * KH * KW + (size_t)(kh * KW + kw)) * parts * I;
        out[base + i] = hi;
        if (split) out[base + I + i] = lo;
    }
}
__global__ void pack_weight_gb16_kernel(const float* __restrict__ wg, const float* __restrict__ wb, uint16_t* __restrict__ out,
                                        int C, int I, int KH, int KW, int BN, int fmt, int split) {
    const long long total = 2LL * C * KH * KW * I;
    const int half = BN / 2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = idx % I;
        long long t = idx / I;
        const int kw = t % KW; t /= KW;
        const int kh = t % KH;
        const int R = t / KH;
        const int tile = R / BN, rr = R % BN;
        const float* src = rr < half ? wg : wb;
        const int c = tile * half + (rr < half ? rr : rr - half);
        uint16_t hi, lo;
        split16(src[(((long long)c * I + i) * KH + kh) * KW + kw], fmt, hi, lo);
        if (!split) {
            out[idx] = hi;
        } else {
            const size_t base = ((size_t)R * KH * KW + (size_t)(kh * KW + kw)) * 2 * I;
            out[base + i] = hi;
            out[base + I + i] = lo;
        }
    }
}

// thin layout: [KH*KW][CinP][Cout]
__global__ void pack_weight_thin_kernel(const float* __restrict__ w, float* __restrict__ out, int O, int I, int CinP,
                                        int KH, int KW) {
    const int total = KH * KW * CinP * O;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const int o = idx % O;
        int t = idx / O;
        const int ci = t % CinP;
        const int tap = t / CinP;
        const int kh = tap / KW, kw = tap % KW;
        out[idx] = ci < I ? w[(((long long)o * I + ci) * KH + kh) * KW + kw] : 0.f;
    }
}

// ------------------------------------------------------------------------------------ thin direct conv
// Block = 8 warps; output tile 8 rows x 16 cols; warp w owns row w, lane owns CPL output channels.
template <int CINP, int CPL>
__global__ void __launch_bounds__(256)
thin_conv_kernel(const mg_thin_args a, int tiles_w, int tiles_h, int num_tiles) {
    extern __shared__ __align__(16) float sm[];
    const int KH = a.KH, KW = a.KW, s = a.stride;
    const int Cout = a.Cout;
    const int PH = 7 * s + KH, PW = 15 * s + KW;  // input patch
    float* w_s = sm;                               // [KH*KW][CINP][Cout]
    float* in_s = sm + KH * KW * CINP * Cout;      // [PH][PW][CINP]
    const int nw = KH * KW * CINP * Cout;
    for (int i = threadIdx.x * 4; i < nw; i += blockDim.x * 4)
        *reinterpret_cast<float4*>(w_s + i) = __ldg(reinterpret_cast<const float4*>(a.w + i));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int R = a.seg_resize > 0 ? a.seg_resize : 1;
    const int IH = a.H, IW = a.W;  // virtual input size (after the nearest resize when seg_resize>0)
    const int c_base = lane * CPL;
    const bool lane_active = c_base < Cout;

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tw = tile % tiles_w;
        const int th = (tile / tiles_w) % tiles_h;
        const int n = tile / (tiles_w * tiles_h);
        const int oh0 = th * 8, ow0 = tw * 16;
        const int ih0 = oh0 * s - a.pad, iw0 = ow0 * s - a.pad;
        __syncthreads();  // previous tile's readers done (also orders the weight fill on the first pass)
        for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
            const int py = i / PW, px = i - py * PW;
            int ih = ih0 + py, iw = iw0 + px;
            bool ok = true;
            if (a.pad_mode == 1) {
                if (ih < 0) ih = -ih;
                if (ih >= IH) ih = 2 * IH - 2 - ih;
                if (iw < 0) iw = -iw;
                if (iw >= IW) iw = 2 * IW - 2 - iw;
                ok = ih >= 0 && ih < IH && iw >= 0 && iw < IW;
            } else {
                ok = ih >= 0 && ih < IH && iw >= 0 && iw < IW;
            }
            float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
            if (ok) {
                const float* src = a.in + (((size_t)n * IH * R + (size_t)ih * R) * ((size_t)IW * R) + (size_t)iw * R) * CINP;
                v0 = __ldg(reinterpret_cast<const float4*>(src));
                if (CINP == 8) v1 = __ldg(reinterpret_cast<const float4*>(src + 4));
            }
            *reinterpret_cast<float4*>(in_s + (size_t)i * CINP) = v0;
            if (CINP == 8) *reinterpret_cast<float4*>(in_s + (size_t)i * CINP + 4) = v1;
        }
        __syncthreads();

        const int oh = oh0 + warp;
#pragma unroll 1
        for (int g = 0; g < 2; ++g) {
            float acc[8][CPL];
#pragma unroll
            for (int p_ = 0; p_ < 8; ++p_)
#pragma unroll
                for (int c = 0; c < CPL; ++c) acc[p_][c] = 0.f;
            if (lane_active) {
                for (int kh = 0; kh < KH; ++kh) {
                    const float* row = in_s + (size_t)((warp * s + kh) * PW) * CINP;
                    for (int kw = 0; kw < KW; ++kw) {
                        const float* wt = w_s + (size_t)((kh * KW + kw) * CINP) * Cout + c_base;
                        float wv[CINP][CPL];
#pragma unroll
                        for (int ci = 0; ci < CINP; ++ci) {
                            if constexpr (CPL == 4) {
                                const float4 t = *reinterpret_cast<const float4*>(wt + (size_t)ci * Cout);
                                wv[ci][0] = t.x; wv[ci][1] = t.y; wv[ci][2] = t.z; wv[ci][3] = t.w;
                            } else {
                                const float2 t = *reinterpret_cast<const float2*>(wt + (size_t)ci * Cout);
                                wv[ci][0] = t.x; wv[ci][1] = t.y;
                            }
                        }
#pragma unroll
                        for (int p_ = 0; p_ < 8; ++p_) {
                            const float* ip = row + (size_t)(((g * 8 + p_) * s + kw)) * CINP;
                            float iv[CINP];
                            const float4 t0 = *reinterpret_cast<const float4*>(ip);
                            iv[0] = t0.x; iv[1] = t0.y; iv[2] = t0.z; iv[3] = t0.w;
                            if constexpr (CINP == 8) {
                                const float4 t1 = *reinterpret_cast<const float4*>(ip + 4);
                                iv[4] = t1.x; iv[5] = t1.y; iv[6] = t1.z; iv[7] = t1.w;
                            }
#pragma unroll
                            for (int ci = 0; ci < CINP; ++ci)
#pragma unroll
                                for (int c = 0; c < CPL; ++c) acc[p_][c] = fmaf(iv[ci], wv[ci][c], acc[p_][c]);
                        }
                    }
                }
            }
            if (lane_active && oh < a.OH) {
                float bv[CPL];
#pragma unroll
                for (int c = 0; c < CPL; ++c) bv[c] = a.bias ? __ldg(a.bias + c_base + c) : 0.f;
#pragma unroll
                for (int p_ = 0; p_ < 8; ++p_) {
                    const int ow = ow0 + g * 8 + p_;
                    if (ow >= a.OW) continue;
                    const size_t pix = ((size_t)n * a.OH + oh) * a.OW + ow;
                    const float ps = a.pscale ? __ldg(a.pscale + pix) : 1.f;
                    const float pm = a.pmul ? __ldg(a.pmul + pix) : 1.f;
                    float y[CPL];
#pragma unroll
                    for (int c = 0; c < CPL; ++c) {
                        float v = act_fn(acc[p_][c] * ps + bv[c], a.act) * pm;
                        y[c] = a.round_out ? rtf32(v) : v;
                    }
                    if (a.out) {
                        float* op = a.out + pix * Cout + c_base;
                        if constexpr (CPL == 4) *reinterpret_cast<float4*>(op) = make_float4(y[0], y[1], y[2], y[3]);
                        else *reinterpret_cast<float2*>(op) = make_float2(y[0], y[1]);
                    }
                    if (a.out_hi) {
                        uint16_t hi[CPL], lo[CPL];
#pragma unroll
                        for (int c = 0; c < CPL; ++c) split16(y[c], a.out16_fmt, hi[c], lo[c]);
                        uint16_t* oh = reinterpret_cast<uint16_t*>(a.out_hi) + pix * Cout + c_base;
                        uint16_t* ol = a.out_lo ? reinterpret_cast<uint16_t*>(a.out_lo) + pix * Cout + c_base : nullptr;
                        if constexpr (CPL == 4) {
                            *reinterpret_cast<uint2*>(oh) = make_uint2(hi[0] | ((uint32_t)hi[1] << 16), hi[2] | ((uint32_t)hi[3] << 16));
                            if (ol) *reinterpret_cast<uint2*>(ol) = make_uint2(lo[0] | ((uint32_t)lo[1] << 16), lo[2] | ((uint32_t)lo[3] << 16));
                        } else {
                            *reinterpret_cast<uint32_t*>(oh) = hi[0] | ((uint32_t)hi[1] << 16);
                            if (ol) *reinterpret_cast<uint32_t*>(ol) = lo[0] | ((uint32_t)lo[1] << 16);
                        }
                    }
                }
            }
        }
    }
}


// ------------------------------------------------------------------------------------ thin conv, register-tiled
// Same contract as thin_conv_kernel, for Cout = 16*CPT (64 or 128): SGEMM-style register tiling, each thread owns
// 8 consecutive pixels of a tile row x CPT channels (tile = 8 rows x 16 cols of pixels, 256 threads = 16 pixel
// groups x 16 channel groups).  Per tap and 4 input channels a thread issues 8 + CPT/ (4/4) shared loads for
// 32*CPT FMAs, i.e. it is FMA-bound rather than LDS-bound.
template <int CINP, int CPT>
__global__ void __launch_bounds__(256, 1)
thin_gemm_kernel(const mg_thin_args a, int tiles_w, int tiles_h, int num_tiles) {
    extern __shared__ __align__(16) float sm[];
    const int KH = a.KH, KW = a.KW, s = a.stride;
    constexpr int Cout = 16 * CPT;
    const int PH = 7 * s + KH, PW = 15 * s + KW;
    float* w_s = sm;                               // [KH*KW][CINP][Cout]
    float* in_s = sm + KH * KW * CINP * Cout;      // [PH][PW][CINP]
    const int nw = KH * KW * CINP * Cout;
    for (int i = threadIdx.x * 4; i < nw; i += blockDim.x * 4)
        *reinterpret_cast<float4*>(w_s + i) = __ldg(reinterpret_cast<const float4*>(a.w + i));
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int prow = ty >> 1, pcol0 = (ty & 1) * 8;
    const int c_base = tx * CPT;
    const int R = a.seg_resize > 0 ? a.seg_resize : 1;
    const int IH = a.H, IW = a.W;
    float bv[CPT];
#pragma unroll
    for (int c = 0; c < CPT; ++c) bv[c] = a.bias ? __ldg(a.bias + c_base + c) : 0.f;

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tw = tile % tiles_w;
        const int th = (tile / tiles_w) % tiles_h;
        const int n = tile / (tiles_w * tiles_h);
        const int oh0 = th * 8, ow0 = tw * 16;
        const int ih0 = oh0 * s - a.pad, iw0 = ow0 * s - a.pad;
        __syncthreads();
        for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
            const int py = i / PW, px = i - py * PW;
            int ih = ih0 + py, iw = iw0 + px;
            if (a.pad_mode == 1) {
                if (ih < 0) ih = -ih;
                if (ih >= IH) ih = 2 * IH - 2 - ih;
                if (iw < 0) iw = -iw;
                if (iw >= IW) iw = 2 * IW - 2 - iw;
            }
            const bool ok = ih >= 0 && ih < IH && iw >= 0 && iw < IW;
            float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
            if (ok) {
                const float* src = a.in + (((size_t)n * IH * R + (size_t)ih * R) * ((size_t)IW * R) + (size_t)iw * R) * CINP;
                v0 = __ldg(reinterpret_cast<const float4*>(src));
                if (CINP == 8) v1 = __ldg(reinterpret_cast<const float4*>(src + 4));
            }
            *reinterpret_cast<float4*>(in_s + (size_t)i * CINP) = v0;
            if (CINP == 8) *reinterpret_cast<float4*>(in_s + (size_t)i * CINP + 4) = v1;
        }
        __syncthreads();

        float acc[8][CPT];
#pragma unroll
        for (int p_ = 0; p_ < 8; ++p_)
#pragma unroll
            for (int c = 0; c < CPT; ++c) acc[p_][c] = 0.f;
        for (int kh = 0; kh < KH; ++kh) {
            const float* row = in_s + (size_t)((prow * s + kh) * PW) * CINP;
            for (int kw = 0; kw < KW; ++kw) {
                const float* wt = w_s + (size_t)((kh * KW + kw) * CINP) * Cout + c_base;
#pragma unroll
                for (int c4 = 0; c4 < CINP; c4 += 4) {
                    float wv[4][CPT];
#pragma unroll
                    for (int ci = 0; ci < 4; ++ci)
#pragma unroll
                        for (int c = 0; c < CPT; c += 4) {
                            const float4 t = *reinterpret_cast<const float4*>(wt + (size_t)(c4 + ci) * Cout + c);
                            wv[ci][c] = t.x; wv[ci][c + 1] = t.y; wv[ci][c + 2] = t.z; wv[ci][c + 3] = t.w;
                        }
#pragma unroll
                    for (int p_ = 0; p_ < 8; ++p_) {
                        const float4 iv = *reinterpret_cast<const float4*>(row + (size_t)((pcol0 + p_) * s + kw) * CINP + c4);
#pragma unroll
                        for (int c = 0; c < CPT; ++c) {
                            acc[p_][c] = fmaf(iv.x, wv[0][c], acc[p_][c]);
                            acc[p_][c] = fmaf(iv.y, wv[1][c], acc[p_][c]);
                            acc[p_][c] = fmaf(iv.z, wv[2][c], acc[p_][c]);
                            acc[p_][c] = fmaf(iv.w, wv[3][c], acc[p_][c]);
                        }
                    }
                }
            }
        }
        const int oh = oh0 + prow;
        if (oh < a.OH) {
#pragma unroll
            for (int p_ = 0; p_ < 8; ++p_) {
                const int ow = ow0 + pcol0 + p_;
                if (ow >= a.OW) continue;
                const size_t pix = ((size_t)n * a.OH + oh) * a.OW + ow;
                const float ps = a.pscale ? __ldg(a.pscale + pix) : 1.f;
                const float pm = a.pmul ? __ldg(a.pmul + pix) : 1.f;
                float y[CPT];
#pragma unroll
                for (int c = 0; c < CPT; ++c) {
                    const float v = act_fn(acc[p_][c] * ps + bv[c], a.act) * pm;
                    y[c] = a.round_out ? rtf32(v) : v;
                }
                if (a.out) {
                    float* op = a.out + pix * Cout + c_base;
#pragma unroll
                    for (int c = 0; c < CPT; c += 4) *reinterpret_cast<float4*>(op + c) = make_float4(y[c], y[c + 1], y[c + 2], y[c + 3]);
                }
                if (a.out_hi) {
                    uint16_t hi[CPT], lo[CPT];
#pragma unroll
                    for (int c = 0; c < CPT; ++c) split16(y[c], a.out16_fmt, hi[c], lo[c]);
                    uint16_t* ohp = reinterpret_cast<uint16_t*>(a.out_hi) + pix * Cout + c_base;
                    uint16_t* olp = a.out_lo ? reinterpret_cast<uint16_t*>(a.out_lo) + pix * Cout + c_base : nullptr;
#pragma unroll
                    for (int c = 0; c < CPT; c += 4) {
                        *reinterpret_cast<uint2*>(ohp + c) = make_uint2(hi[c] | ((uint32_t)hi[c + 1] << 16), hi[c + 2] | ((uint32_t)hi[c + 3] << 16));
                        if (olp) *reinterpret_cast<uint2*>(olp + c) = make_uint2(lo[c] | ((uint32_t)lo[c + 1] << 16), lo[c + 2] | ((uint32_t)lo[c + 3] << 16));
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------ conv_img (Cin -> 3, NCHW out)
// tile 8 x 32 pixels per block (256 threads, one pixel each); input tile staged as [c4][pixel][4].
__global__ void __launch_bounds__(256)
conv_img_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                float* __restrict__ out, int N, int H, int W, int Cin, int Cout, int act_in, int act_out) {
    extern __shared__ __align__(16) float sm[];
    const int PW = 34, PH = 10, NP = PW * PH;
    const int C4 = Cin / 4;
    float* in_s = sm;                      // [C4][NP][4]
    float* w_s = sm + (size_t)C4 * NP * 4; // [9][Cin][4]  (co padded to 4)
    for (int i = threadIdx.x; i < 9 * Cin * 4; i += blockDim.x) {
        const int co = i & 3;
        const int ci = (i >> 2) % Cin;
        const int tap = (i >> 2) / Cin;
        w_s[i] = co < Cout ? w[((size_t)co * Cin + ci) * 9 + tap] : 0.f;
    }
    const int tiles_w = (W + 31) / 32, tiles_h = (H + 7) / 8;
    const int tile = blockIdx.x;
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
    const int h0 = th * 8 - 1, w0 = tw * 32 - 1;
    // coalesced fill: consecutive threads read consecutive float4 of one pixel; four independent loads in flight per thread
    // (87 KB per block through 256 threads with one load each was 21 serial L2/DRAM round trips)
    for (int i0 = threadIdx.x; i0 < NP * C4; i0 += 4 * blockDim.x) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + u * blockDim.x;
            const int c4 = i % C4, pp = i / C4;
            const int py = pp / PW, px = pp - py * PW;
            const int ih = h0 + py, iw = w0 + px;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < NP * C4 && ih >= 0 && ih < H && iw >= 0 && iw < W)
                v[u] = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H + ih) * W + iw) * Cin) + c4);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + u * blockDim.x;
            if (i >= NP * C4) break;
            const int c4 = i % C4, pp = i / C4;
            // act_fn(0) == 0 for every activation used here, so the padding stays zero
            const float4 r = make_float4(act_fn(v[u].x, act_in), act_fn(v[u].y, act_in), act_fn(v[u].z, act_in), act_fn(v[u].w, act_in));
            *reinterpret_cast<float4*>(in_s + ((size_t)c4 * NP + pp) * 4) = r;
        }
    }
    __syncthreads();
    const int ly = threadIdx.x >> 5, lx = threadIdx.x & 31;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            const int pp = (ly + kh) * PW + lx + kw;
            const float* wt = w_s + (size_t)((kh * 3 + kw) * Cin) * 4;
#pragma unroll 4
            for (int c4 = 0; c4 < C4; ++c4) {
                const float4 v = *reinterpret_cast<const float4*>(in_s + ((size_t)c4 * NP + pp) * 4);
                const float4 w0v = *reinterpret_cast<const float4*>(wt + (c4 * 4 + 0) * 4);
                const float4 w1v = *reinterpret_cast<const float4*>(wt + (c4 * 4 + 1) * 4);
                const float4 w2v = *reinterpret_cast<const float4*>(wt + (c4 * 4 + 2) * 4);
                const float4 w3v = *reinterpret_cast<const float4*>(wt + (c4 * 4 + 3) * 4);
                a0 = fmaf(v.x, w0v.x, a0); a1 = fmaf(v.x, w0v.y, a1); a2 = fmaf(v.x, w0v.z, a2);
                a0 = fmaf(v.y, w1v.x, a0); a1 = fmaf(v.y, w1v.y, a1); a2 = fmaf(v.y, w1v.z, a2);
                a0 = fmaf(v.z, w2v.x, a0); a1 = fmaf(v.z, w2v.y, a1); a2 = fmaf(v.z, w2v.z, a2);
                a0 = fmaf(v.w, w3v.x, a0); a1 = fmaf(v.w, w3v.y, a1); a2 = fmaf(v.w, w3v.z, a2);
            }
        }
    const int oh = th * 8 + ly, ow = tw * 32 + lx;
    if (oh < H && ow < W) {
        const float r[3] = {a0, a1, a2};
        for (int co = 0; co < Cout; ++co)
            out[(((size_t)n * Cout + co) * H + oh) * W + ow] = act_fn(r[co] + (bias ? bias[co] : 0.f), act_out);
    }
}

// ------------------------------------------------------------------------------------ Cin -> 1 conv (PatchGAN logits)
__global__ void __launch_bounds__(256)
conv_to1_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                float* __restrict__ out, int N, int H, int W, int Cin, int KH, int KW, int pad, int OH, int OW) {
    extern __shared__ __align__(16) float w_s[];  // [KH*KW][Cin]
    for (int i = threadIdx.x; i < KH * KW * Cin; i += blockDim.x) {
        const int ci = i % Cin, tap = i / Cin;
        w_s[i] = w[(size_t)ci * KH * KW + tap];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long total = (long long)N * OH * OW;
    for (long long o = blockIdx.x * 8LL + warp; o < total; o += gridDim.x * 8LL) {
        const int ow = o % OW;
        const int oh = (o / OW) % OH;
        const int n = o / ((long long)OW * OH);
        float acc = 0.f;
        for (int kh = 0; kh < KH; ++kh) {
            const int ih = oh + kh - pad;
            if (ih < 0 || ih >= H) continue;
            for (int kw = 0; kw < KW; ++kw) {
                const int iw = ow + kw - pad;
                if (iw < 0 || iw >= W) continue;
                const float4* xp = reinterpret_cast<const float4*>(x + (((size_t)n * H + ih) * W + iw) * Cin);
                const float4* wp = reinterpret_cast<const float4*>(w_s + (size_t)(kh * KW + kw) * Cin);
                for (int c4 = lane; c4 < Cin / 4; c4 += 32) {
                    const float4 a = __ldg(xp + c4);
                    const float4 b = wp[c4];
                    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
                    acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
                }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
        if (lane == 0) out[o] = acc + (bias ? bias[0] : 0.f);
    }
}

// ------------------------------------------------------------------------------------ per-channel statistics
// x viewed as [B][P][C]; sums [B][2][C] doubles.  Threads along channels (float4), rows of threads
// stride over pixels; fp32 partials are flushed to double every 32 pixels; warp-free smem reduce,
// one double atomic per (block, channel, moment).
__global__ void __launch_bounds__(256, 3)
chan_stats_kernel(const float* __restrict__ x, long long P, int C, double* __restrict__ sums, int blocks_per_b,
                  uint16_t* __restrict__ out16) {
    const int G = C / 4;                    // float4 groups
    const int tpr = G < 256 ? G : 256;      // threads per pixel row
    const int rows = 256 / tpr;
    const int b = blockIdx.x / blocks_per_b;
    const int blk = blockIdx.x % blocks_per_b;
    const int tr = threadIdx.x / tpr, tc = threadIdx.x % tpr;
    const float* xb = x + (size_t)b * P * C;
    double* sb = sums + (size_t)b * 2 * C;
    __shared__ double red[256 * 8];
    for (int g0 = tc; g0 < G; g0 += tpr) {
        double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
        float fs[4] = {0, 0, 0, 0}, fq[4] = {0, 0, 0, 0};
        int cnt = 0;
        if (threadIdx.x < rows * tpr) {
            auto add = [&](const float4 v, long long pidx) {
                if (out16) {   // bf16 copy in the same pass (operand of the 16-bit gradient GEMMs; B == 1 only)
                    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), bb = __floats2bfloat162_rn(v.z, v.w);
                    *reinterpret_cast<uint2*>(out16 + (size_t)pidx * C + g0 * 4) =
                        make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&bb));
                }
                fs[0] += v.x; fs[1] += v.y; fs[2] += v.z; fs[3] += v.w;
                fq[0] = fmaf(v.x, v.x, fq[0]); fq[1] = fmaf(v.y, v.y, fq[1]);
                fq[2] = fmaf(v.z, v.z, fq[2]); fq[3] = fmaf(v.w, v.w, fq[3]);
                if (++cnt == 32) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) { s[i] += fs[i]; q[i] += fq[i]; fs[i] = 0.f; fq[i] = 0.f; }
                    cnt = 0;
                }
            };
            // four independent loads in flight per thread (one was 60 % of the HBM rate: 32 warps x 512 B per SM does not cover
            // the DRAM latency); the accumulation order, and with it every bit of the result, is unchanged
            const long long step = (long long)blocks_per_b * rows;
            long long pidx = (long long)blk * rows + tr;
            for (; pidx + 3 * step < P; pidx += 4 * step) {
                float4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(xb + (size_t)(pidx + u * step) * C) + g0);
#pragma unroll
                for (int u = 0; u < 4; ++u) add(v[u], pidx + u * step);
            }
            for (; pidx < P; pidx += step) add(__ldg(reinterpret_cast<const float4*>(xb + (size_t)pidx * C) + g0), pidx);
#pragma unroll
            for (int i = 0; i < 4; ++i) { s[i] += fs[i]; q[i] += fq[i]; }
        }
        if (rows > 1) {
            __syncthreads();
#pragma unroll
            for (int i = 0; i < 4; ++i) { red[threadIdx.x * 8 + i] = s[i]; red[threadIdx.x * 8 + 4 + i] = q[i]; }
            __syncthreads();
            if (tr == 0) {
                for (int r = 1; r < rows; ++r)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        s[i] += red[(r * tpr + tc) * 8 + i];
                        q[i] += red[(r * tpr + tc) * 8 + 4 + i];
                    }
            }
        }
        if (tr == 0 && threadIdx.x < rows * tpr) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                atomicAdd(sb + g0 * 4 + i, s[i]);
                atomicAdd(sb + C + g0 * 4 + i, q[i]);
            }
        }
    }
}

// count <= 0: the sample count is the (all-reduced) element sums[2*C] - the per-replica sum_size summed over ranks
// (batchnorm.py:119), so uneven shards stay exact; unb_mult = 4^s for a folded 2^s nearest upsample.
__global__ void bn_finalize_kernel(const double* __restrict__ sums, int C, double count, double unb_mult, float eps,
                                   float momentum, int clamp_mode, float* nscale, float* nshift, float* rmean,
                                   float* rvar, float* mean_out, float* var_out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    if (count <= 0.0) count = sums[2 * C];
    const double count_u = count * unb_mult;
    const double mean = sums[c] / count;
    double var = sums[C + c] / count - mean * mean;
    if (var < 0) var = 0;
    double rstd;
    if (clamp_mode == 1) rstd = 1.0 / sqrt(var < (double)eps ? (double)eps : var);
    else rstd = 1.0 / sqrt(var + (double)eps);
    nscale[c] = (float)rstd;
    nshift[c] = (float)(-mean * rstd);
    if (mean_out) mean_out[c] = (float)mean;
    if (var_out) var_out[c] = (float)var;
    // batchnorm.py:139-143 as eager fp32 ops: (1 - m) * running + m * stat, both products rounded before the add
    if (rmean) rmean[c] = __fadd_rn(__fmul_rn(1.f - momentum, rmean[c]), __fmul_rn(momentum, (float)mean));
    if (rvar) {
        const double unb = count_u > 1.0 ? var * count_u / (count_u - 1.0) : var;
        rvar[c] = __fadd_rn(__fmul_rn(1.f - momentum, rvar[c]), __fmul_rn(momentum, (float)unb));
    }
}

__global__ void bn_from_running_kernel(const float* rmean, const float* rvar, int C, float eps, float* nscale,
                                       float* nshift) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float rstd = 1.f / sqrtf(rvar[c] + eps);
    nscale[c] = rstd;
    nshift[c] = -rmean[c] * rstd;
}

// InstanceNorm: sums [N][2][C] doubles -> ss [N][2][C] floats (rstd, -mean*rstd)
__global__ void in_finalize_kernel(const double* __restrict__ sums, float* __restrict__ ss, int N, int C, double HW,
                                   float eps) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * C) return;
    const int n = idx / C, c = idx % C;
    const double mean = sums[(size_t)n * 2 * C + c] / HW;
    double var = sums[(size_t)n * 2 * C + C + c] / HW - mean * mean;
    if (var < 0) var = 0;
    const double rstd = 1.0 / sqrt(var + (double)eps);
    ss[(size_t)n * 2 * C + c] = (float)rstd;
    ss[(size_t)n * 2 * C + C + c] = (float)(-mean * rstd);
}
// InstanceNorm apply: x [N][HW][C], ss [N][2][C]
__global__ void in_apply_kernel(const float* __restrict__ x, const float* __restrict__ ss, float* __restrict__ y,
                                int N, long long HW, int C, int act, int round_, const float* __restrict__ pmul,
                                uint16_t* __restrict__ y_hi, uint16_t* __restrict__ y_lo, int fmt16) {
    const int G = C / 4;
    const long long total = (long long)N * HW * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g = idx % G;
        const long long pix = idx / G;
        const int n = pix / HW;
        const float* sb = ss + (size_t)n * 2 * C;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + idx);
        const float4 sc = __ldg(reinterpret_cast<const float4*>(sb) + g);
        const float4 sh = __ldg(reinterpret_cast<const float4*>(sb + C) + g);
        float r[4] = {fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w)};
        const float pm = pmul ? __ldg(pmul + pix) : 1.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float t = act_fn(r[i], act) * pm;
            r[i] = round_ ? rtf32(t) : t;
        }
        if (y) reinterpret_cast<float4*>(y)[idx] = make_float4(r[0], r[1], r[2], r[3]);
        if (y_hi) {
            uint16_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split16(r[i], fmt16, hi[i], lo[i]);
            reinterpret_cast<uint2*>(y_hi)[idx] = make_uint2(hi[0] | ((uint32_t)hi[1] << 16), hi[2] | ((uint32_t)hi[3] << 16));
            if (y_lo) reinterpret_cast<uint2*>(y_lo)[idx] = make_uint2(lo[0] | ((uint32_t)lo[1] << 16), lo[2] | ((uint32_t)lo[3] << 16));
        }
    }
}

// ------------------------------------------------------------------------------------ input preparation
__global__ void prep_seg_kernel(const float* __restrict__ tag, const float* __restrict__ orient, int oc,
                                float* __restrict__ seg4, int N, long long HW) {
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int n = idx / HW;
        const long long p = idx - (long long)n * HW;
        const float t0 = tag[((size_t)n * 2 + 0) * HW + p];
        const float t1 = tag[((size_t)n * 2 + 1) * HW + p];
        float o0, o1;
        if (oc == 1) {
            // generator.py:131-133: orient/255*pi, [sin 2th, cos 2th] * hair
            const float th = orient[(size_t)n * HW + p] / 255.0f * 3.14159265358979323846f;
            o0 = sinf(2.f * th) * t1;
            o1 = cosf(2.f * th) * t1;
        } else {
            o0 = orient[((size_t)n * 2 + 0) * HW + p];
            o1 = orient[((size_t)n * 2 + 1) * HW + p];
        }
        reinterpret_cast<float4*>(seg4)[idx] = make_float4(t0, t1, o0, o1);
    }
}

__global__ void prep_dinput_kernel(const float* __restrict__ seg4, const float* __restrict__ img,
                                   float* __restrict__ out8, int N, long long HW) {
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int n = idx / HW;
        const long long p = idx - (long long)n * HW;
        const float4 s = __ldg(reinterpret_cast<const float4*>(seg4) + idx);
        const float r = img[((size_t)n * 3 + 0) * HW + p];
        const float g = img[((size_t)n * 3 + 1) * HW + p];
        const float b = img[((size_t)n * 3 + 2) * HW + p];
        float4* o = reinterpret_cast<float4*>(out8) + idx * 2;
        o[0] = s;
        o[1] = make_float4(r, g, b, 0.f);
    }
}

__global__ void prep_bginput_kernel(const float* __restrict__ img, const float* __restrict__ noise,
                                    const float* __restrict__ back, float* __restrict__ out4, int N, long long HW) {
    const long long total = (long long)N * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int n = idx / HW;
        const long long p = idx - (long long)n * HW;
        const float bm = back[idx];
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t o = ((size_t)n * 3 + c) * HW + p;
            v[c] = __fadd_rn(__fmul_rn(img[o], bm), __fmul_rn(noise[o], 1.f - bm));   // encoder.py:321's eager order
        }
        reinterpret_cast<float4*>(out4)[idx] = make_float4(v[0], v[1], v[2], 0.f);
    }
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int C, long long HW,
                                    int CP, const float* __restrict__ pmul) {
    const long long total = (long long)N * HW * CP;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = idx % CP;
        const long long pix = idx / CP;
        const int n = pix / HW;
        const long long p = pix - (long long)n * HW;
        out[idx] = c < C ? in[((size_t)n * C + c) * HW + p] * (pmul ? pmul[pix] : 1.f) : 0.f;
    }
}

// PartialConv2d mask bookkeeping (partialconv2d.py:57-66), single-channel mask [N,H,W]:
// um = sum of mask over the k x k window (zero padded); ratio = k*k/(um+1e-8)*clamp(um,0,1); update = clamp(um,0,1).
// The reference's `slide_winsize / t` is a Python float over a tensor, which torch evaluates as t.reciprocal() * slide_winsize.
__global__ void partial_mask_kernel(const float* __restrict__ mask, float* __restrict__ ratio, float* __restrict__ update,
                                    int N, int H, int W, int OH, int OW, int k, int s, int p) {
    const long long total = (long long)N * OH * OW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int ow = idx % OW;
        const int oh = (idx / OW) % OH;
        const int n = idx / ((long long)OW * OH);
        float um = 0.f;
        for (int kh = 0; kh < k; ++kh) {
            const int ih = oh * s + kh - p;
            if (ih < 0 || ih >= H) continue;
            for (int kw = 0; kw < k; ++kw) {
                const int iw = ow * s + kw - p;
                if (iw < 0 || iw >= W) continue;
                um += mask[((size_t)n * H + ih) * W + iw];
            }
        }
        const float r = __fmul_rn(__frcp_rn(um + 1e-8f), (float)(k * k));
        const float u = fminf(fmaxf(um, 0.f), 1.f);
        ratio[idx] = r * u;
        update[idx] = u;
    }
}

// ImageEncoder3 tail (encoder.py:207-220): per sample, mean of x over the reference-hair pixels
// (sum / max(count,1)), broadcast onto the target-hair pixels.  Masks are full-resolution [N,MH,MW]
// read through the legacy nearest resize (index * MH/h).  One block per (n, 32-channel group).
__global__ void masked_mean_bcast_kernel(const float* __restrict__ x, const float* __restrict__ mref,
                                         const float* __restrict__ mtag, float* __restrict__ out, int N, int h, int w,
                                         int C, int MH, int MW) {
    const int n = blockIdx.y;
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int row = threadIdx.x >> 5;  // 8 rows of threads stride over pixels
    const int sh = MH / h, sw = MW / w;
    __shared__ float red[8][33];
    __shared__ float cnt_s[8];
    float acc = 0.f, cnt = 0.f;
    for (int pidx = row; pidx < h * w; pidx += 8) {
        const int ph = pidx / w, pw = pidx - ph * w;
        const float m = mref[((size_t)n * MH + (size_t)ph * sh) * MW + (size_t)pw * sw];
        cnt += m;
        if (c < C) acc += x[(((size_t)n * h + ph) * w + pw) * C + c] * m;
    }
    red[row][threadIdx.x & 31] = acc;
    if ((threadIdx.x & 31) == 0) cnt_s[row] = cnt;
    __syncthreads();
    float tot = 0.f, ctot = 0.f;
    for (int r = 0; r < 8; ++r) { tot += red[r][threadIdx.x & 31]; ctot += cnt_s[r]; }
    const float mean = tot / fmaxf(ctot, 1.f);
    for (int pidx = row; pidx < h * w; pidx += 8) {
        const int ph = pidx / w, pw = pidx - ph * w;
        const float m = mtag[((size_t)n * MH + (size_t)ph * sh) * MW + (size_t)pw * sw];
        if (c < C) out[(((size_t)n * h + ph) * w + pw) * C + c] = mean * m;
    }
}

// F.interpolate(mode='bilinear', align_corners=False) on NHWC (encoder.py:222-223)
__global__ void resize_bilinear_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C,
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
        const float ly = fy - y0, lx = fx - x0;
        const float* b = in + (size_t)n * H * W * C + c;
        const float v00 = b[((size_t)y0 * W + x0) * C], v01 = b[((size_t)y0 * W + x1) * C];
        const float v10 = b[((size_t)y1 * W + x0) * C], v11 = b[((size_t)y1 * W + x1) * C];
        out[idx] = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
    }
}

// ReflectionPad2d(p) on NHWC, optional TF32 rounding (MaskGAN_networks.py:120-121,168)
__global__ void reflect_pad_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C, int p,
                                   int round_, uint16_t* __restrict__ o_hi, uint16_t* __restrict__ o_lo, int fmt16) {
    const int G = C / 4;
    const int PH = H + 2 * p, PW = W + 2 * p;
    const long long total = (long long)N * PH * PW * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g = idx % G;
        long long t = idx / G;
        const int pw = t % PW; t /= PW;
        const int ph = t % PH;
        const int n = t / PH;
        int ih = ph - p, iw = pw - p;
        if (ih < 0) ih = -ih;
        if (ih >= H) ih = 2 * H - 2 - ih;
        if (iw < 0) iw = -iw;
        if (iw >= W) iw = 2 * W - 2 - iw;
        float4 v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)n * H + ih) * W + iw) * C) + g);
        if (round_) { v.x = rtf32(v.x); v.y = rtf32(v.y); v.z = rtf32(v.z); v.w = rtf32(v.w); }
        if (out) reinterpret_cast<float4*>(out)[idx] = v;
        if (o_hi) {
            const float r[4] = {v.x, v.y, v.z, v.w};
            uint16_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split16(r[i], fmt16, hi[i], lo[i]);
            reinterpret_cast<uint2*>(o_hi)[idx] = make_uint2(hi[0] | ((uint32_t)hi[1] << 16), hi[2] | ((uint32_t)hi[3] << 16));
            if (o_lo) reinterpret_cast<uint2*>(o_lo)[idx] = make_uint2(lo[0] | ((uint32_t)lo[1] << 16), lo[2] | ((uint32_t)lo[3] << 16));
        }
    }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int C, long long HW,
                                    int CP) {
    const long long total = (long long)N * C * HW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long p = idx % HW;
        const int c = (idx / HW) % C;
        const int n = idx / (HW * C);
        out[idx] = in[((size_t)n * HW + p) * CP + c];
    }
}

// separable max filter on [N,H,W]; dir 0: along W, dir 1: along H
__global__ void maxfilt_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int k, int dir,
                               int invert) {
    const long long total = (long long)N * H * W;
    const int p = k / 2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int w = idx % W;
        const int h = (idx / W) % H;
        const long long base = idx - (dir == 0 ? w : (long long)h * W);
        float m = -INFINITY;
        if (dir == 0) {
            for (int j = w - p; j <= w - p + k - 1; ++j)
                if (j >= 0 && j < W) m = fmaxf(m, in[base + j]);
        } else {
            for (int j = h - p; j <= h - p + k - 1; ++j)
                if (j >= 0 && j < H) m = fmaxf(m, in[base + (long long)j * W]);
        }
        out[idx] = invert ? 1.f - m : m;
    }
}

__global__ void avgpool3s2_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C,
                                  int OH, int OW) {
    const int G = C / 4;
    const long long total = (long long)N * OH * OW * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int g = idx % G;
        long long t = idx / G;
        const int ow = t % OW; t /= OW;
        const int oh = t % OH;
        const int n = t / OH;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        int cnt = 0;
        for (int dh = -1; dh <= 1; ++dh) {
            const int ih = oh * 2 + dh;
            if (ih < 0 || ih >= H) continue;
            for (int dw = -1; dw <= 1; ++dw) {
                const int iw = ow * 2 + dw;
                if (iw < 0 || iw >= W) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)n * H + ih) * W + iw) * C) + g);
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                ++cnt;
            }
        }
        const float inv = 1.f / (float)cnt;
        reinterpret_cast<float4*>(out)[idx] = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
    }
}

static int ew_grid(long long total, int block = 256) {
    long long g = (total + block - 1) / block;
    const long long cap = (long long)num_sms() * 16;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace mg

using namespace mg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mg_pack_weight(const float* w, float* wpack, int O, int I, int KH, int KW, const float* inv_sigma,
                              int round_tf32, void* stream) {
    if (!w || !wpack) return set_error(-1, "mg_pack_weight: null pointer");
    const long long total = (long long)O * I * KH * KW;
    pack_weight_kernel<<<ew_grid(total), 256, 0, ST(stream)>>>(w, wpack, O, I, KH, KW, inv_sigma, round_tf32);
    return check_launch("mg_pack_weight");
}
extern "C" int mg_pack_weight_gb(const float* wg, const float* wb, float* wpack, int C, int I, int KH, int KW, int BN,
                                 void* stream) {
    if (!wg || !wb || !wpack) return set_error(-1, "mg_pack_weight_gb: null pointer");
    if (BN % 64 != 0 || (2 * C) % BN != 0) return set_error(-2, "mg_pack_weight_gb: bad BN %d for C %d", BN, C);
    const long long total = 2LL * C * I * KH * KW;
    pack_weight_gb_kernel<<<ew_grid(total), 256, 0, ST(stream)>>>(wg, wb, wpack, C, I, KH, KW, BN);
    return check_launch("mg_pack_weight_gb");
}
extern "C" int mg_pack_weight_thin(const float* w, float* wt, int O, int I, int CinP, int KH, int KW, void* stream) {
    if (!w || !wt) return set_error(-1, "mg_pack_weight_thin: null pointer");
    if (I > CinP) return set_error(-2, "mg_pack_weight_thin: I %d > CinP %d", I, CinP);
    pack_weight_thin_kernel<<<ew_grid((long long)KH * KW * CinP * O), 256, 0, ST(stream)>>>(w, wt, O, I, CinP, KH, KW);
    return check_launch("mg_pack_weight_thin");
}

extern "C" int mg_conv_thin(const mg_thin_args* a, void* stream) {
    if (!a || !a->in || !a->w || (!a->out && !a->out_hi)) return set_error(-1, "mg_conv_thin: null pointer");
    if (a->out_hi && (a->out16_fmt < 1 || a->out16_fmt > 2)) return set_error(-6, "mg_conv_thin: out16_fmt must be 1 or 2");
    if (a->CinP != 4 && a->CinP != 8) return set_error(-2, "mg_conv_thin: CinP must be 4 or 8");
    if (a->Cout % 32 != 0 || a->Cout > 128) return set_error(-3, "mg_conv_thin: Cout %d unsupported (multiple of 32, <=128)", a->Cout);
    if (a->seg_resize > 0 && a->CinP != 4) return set_error(-4, "mg_conv_thin: seg_resize needs CinP 4");
    const int cpl = a->Cout > 64 ? 4 : 2;
    const int tiles_w = cdiv(a->OW, 16), tiles_h = cdiv(a->OH, 8);
    const int num_tiles = tiles_w * tiles_h * a->N;
    const int PH = 7 * a->stride + a->KH, PW = 15 * a->stride + a->KW;
    const size_t smem = ((size_t)a->KH * a->KW * a->CinP * a->Cout + (size_t)PH * PW * a->CinP) * 4;
    if (smem > 200 * 1024) return set_error(-5, "mg_conv_thin: smem %zu too large", smem);
    int grid = num_sms() * 2;
    if (grid > num_tiles) grid = num_tiles;
#define LAUNCH_THIN(CI, CP)                                                                                  \
    do {                                                                                                     \
        cudaError_t e = cudaFuncSetAttribute(thin_conv_kernel<CI, CP>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                             200 * 1024);                                                    \
        if (e != cudaSuccess) return set_error((int)e, "thin attr: %s", cudaGetErrorString(e));              \
        thin_conv_kernel<CI, CP><<<grid, 256, smem, ST(stream)>>>(*a, tiles_w, tiles_h, num_tiles);          \
    } while (0)
    const int use_gemm = tune(TK_THIN_GEMM);
    // the register-tiled variant serves Cout = 64 (k7 / k4 layers), the lane-per-channel one Cout = 128
    if ((use_gemm == 2 && a->Cout == 128) || (use_gemm >= 1 && a->Cout == 64)) {
#define LAUNCH_TG(CI, CT)                                                                                     \
    do {                                                                                                      \
        cudaError_t e = cudaFuncSetAttribute(thin_gemm_kernel<CI, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                             200 * 1024);                                                     \
        if (e != cudaSuccess) return set_error((int)e, "thin attr: %s", cudaGetErrorString(e));               \
        int g1 = num_sms() * (CT == 8 ? 1 : 2); if (g1 > num_tiles) g1 = num_tiles;                                            \
        thin_gemm_kernel<CI, CT><<<g1, 256, smem, ST(stream)>>>(*a, tiles_w, tiles_h, num_tiles);             \
    } while (0)
        if (a->CinP == 4 && a->Cout == 128) LAUNCH_TG(4, 8);
        else if (a->CinP == 4) LAUNCH_TG(4, 4);
        else if (a->Cout == 128) LAUNCH_TG(8, 8);
        else LAUNCH_TG(8, 4);
        return check_launch("mg_conv_thin");
    }
    if (a->CinP == 4 && cpl == 4) LAUNCH_THIN(4, 4);
    else if (a->CinP == 4) LAUNCH_THIN(4, 2);
    else if (cpl == 4) LAUNCH_THIN(8, 4);
    else LAUNCH_THIN(8, 2);
    return check_launch("mg_conv_thin");
}

extern "C" int mg_conv_img(const float* x, const float* w, const float* bias, float* out, int N, int H, int W, int Cin,
                           int Cout, int act_in, int act_out, void* stream) {
    if (!x || !w || !out) return set_error(-1, "mg_conv_img: null pointer");
    if (Cin % 4 != 0 || Cout > 3) return set_error(-2, "mg_conv_img: Cin%%4==0 and Cout<=3 required");
    const size_t smem = ((size_t)(Cin / 4) * 340 * 4 + (size_t)9 * Cin * 4) * 4;
    if (smem > 200 * 1024) return set_error(-3, "mg_conv_img: Cin %d too large", Cin);
    cudaError_t e = cudaFuncSetAttribute(conv_img_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return set_error((int)e, "conv_img attr: %s", cudaGetErrorString(e));
    const int tiles = cdiv(W, 32) * cdiv(H, 8) * N;
    conv_img_kernel<<<tiles, 256, smem, ST(stream)>>>(x, w, bias, out, N, H, W, Cin, Cout, act_in, act_out);
    return check_launch("mg_conv_img");
}

extern "C" int mg_conv_to1(const float* x, const float* w, const float* bias, float* out, int N, int H, int W, int Cin,
                           int KH, int KW, int pad, void* stream) {
    if (!x || !w || !out) return set_error(-1, "mg_conv_to1: null pointer");
    if (Cin % 4 != 0) return set_error(-2, "mg_conv_to1: Cin%%4");
    const int OH = H + 2 * pad - KH + 1, OW = W + 2 * pad - KW + 1;
    const size_t smem = (size_t)KH * KW * Cin * 4;
    cudaError_t e = cudaFuncSetAttribute(conv_to1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return set_error((int)e, "conv_to1 attr: %s", cudaGetErrorString(e));
    const long long total = (long long)N * OH * OW;
    int grid = (int)((total + 7) / 8);
    const int cap = num_sms() * 4;
    if (grid > cap) grid = cap;
    conv_to1_kernel<<<grid, 256, smem, ST(stream)>>>(x, w, bias, out, N, H, W, Cin, KH, KW, pad, OH, OW);
    return check_launch("mg_conv_to1");
}

static int launch_stats(const float* x, int B, long long P, int C, double* sums, cudaStream_t st, uint16_t* out16 = nullptr) {
    if (C % 4 != 0 || C > 4096 || (C > 1024 && C % 1024 != 0)) return set_error(-2, "chan_stats: C %d unsupported", C);
    const int G = C / 4;
    const int tpr = G < 256 ? G : 256;
    const int rows = 256 / tpr;
    long long want = (P + (long long)rows * 8 - 1) / ((long long)rows * 8);
    long long cap = ((long long)num_sms() * 3 + B - 1) / B;   // 3 resident blocks per SM (80 registers): one wave
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    chan_stats_kernel<<<(int)want * B, 256, 0, st>>>(x, P, C, sums, (int)want, out16);
    return check_launch("chan_stats");
}
extern "C" int mg_bn_stats(const float* x, long long P, int C, double* sums, void* stream) {
    if (!x || !sums) return set_error(-1, "mg_bn_stats: null pointer");
    return launch_stats(x, 1, P, C, sums, ST(stream));
}
extern "C" int mg_bn_stats_cvt16(const float* x, long long P, int C, double* sums, void* out_bf16, void* stream) {
    if (!x || !sums || !out_bf16) return set_error(-1, "mg_bn_stats_cvt16: null pointer");
    return launch_stats(x, 1, P, C, sums, ST(stream), static_cast<uint16_t*>(out_bf16));
}
extern "C" int mg_in_stats(const float* x, int N, long long HW, int C, double* sums, void* stream) {
    if (!x || !sums) return set_error(-1, "mg_in_stats: null pointer");
    return launch_stats(x, N, HW, C, sums, ST(stream));
}
extern "C" int mg_bn_finalize(const double* sums, int C, double count, double unbiased_mult, float eps, float momentum,
                              int clamp_mode, float* nscale, float* nshift, float* running_mean, float* running_var,
                              float* mean_out, float* var_out, void* stream) {
    if (!sums || !nscale || !nshift) return set_error(-1, "mg_bn_finalize: null pointer");
    if (unbiased_mult < 1.0) return set_error(-2, "mg_bn_finalize: unbiased_mult must be >= 1");
    bn_finalize_kernel<<<cdiv(C, 128), 128, 0, ST(stream)>>>(sums, C, count, unbiased_mult, eps, momentum, clamp_mode,
                                                             nscale, nshift, running_mean, running_var, mean_out, var_out);
    return check_launch("mg_bn_finalize");
}
extern "C" int mg_bn_from_running(const float* rm, const float* rv, int C, float eps, float* nscale, float* nshift,
                                  void* stream) {
    if (!rm || !rv || !nscale || !nshift) return set_error(-1, "mg_bn_from_running: null pointer");
    bn_from_running_kernel<<<cdiv(C, 128), 128, 0, ST(stream)>>>(rm, rv, C, eps, nscale, nshift);
    return check_launch("mg_bn_from_running");
}
extern "C" int mg_in_apply(const float* x, const double* sums, float* ss, float* y, int N, long long HW, int C, float eps,
                           int act, int round_out, const float* pmul, void* y_hi, void* y_lo, int out16_fmt, void* stream) {
    if (!x || !sums || (!y && !y_hi) || !ss) return set_error(-1, "mg_in_apply: null pointer");
    if (y_hi && (out16_fmt < 1 || out16_fmt > 2)) return set_error(-3, "mg_in_apply: out16_fmt must be 1 or 2");
    if (C % 4 != 0) return set_error(-2, "mg_in_apply: C%%4");
    in_finalize_kernel<<<cdiv((long long)N * C, 128), 128, 0, ST(stream)>>>(sums, ss, N, C, (double)HW, eps);
    count_launch();
    in_apply_kernel<<<ew_grid((long long)N * HW * (C / 4)), 256, 0, ST(stream)>>>(x, ss, y, N, HW, C, act, round_out, pmul,
                                                                                 (uint16_t*)y_hi, (uint16_t*)y_lo, out16_fmt);
    return check_launch("mg_in_apply");
}

extern "C" int mg_prep_seg(const float* tag, const float* orient, int oc, float* seg4, int N, int H, int W, void* stream) {
    if (!tag || !orient || !seg4) return set_error(-1, "mg_prep_seg: null pointer");
    if (oc != 1 && oc != 2) return set_error(-2, "mg_prep_seg: orient channels must be 1 or 2");
    prep_seg_kernel<<<ew_grid((long long)N * H * W), 256, 0, ST(stream)>>>(tag, orient, oc, seg4, N, (long long)H * W);
    return check_launch("mg_prep_seg");
}
extern "C" int mg_prep_dinput(const float* seg4, const float* img, float* out8, int N, int H, int W, void* stream) {
    if (!seg4 || !img || !out8) return set_error(-1, "mg_prep_dinput: null pointer");
    prep_dinput_kernel<<<ew_grid((long long)N * H * W), 256, 0, ST(stream)>>>(seg4, img, out8, N, (long long)H * W);
    return check_launch("mg_prep_dinput");
}
extern "C" int mg_prep_bginput(const float* img, const float* noise, const float* back, float* out4, int N, int H, int W,
                               void* stream) {
    if (!img || !noise || !back || !out4) return set_error(-1, "mg_prep_bginput: null pointer");
    prep_bginput_kernel<<<ew_grid((long long)N * H * W), 256, 0, ST(stream)>>>(img, noise, back, out4, N, (long long)H * W);
    return check_launch("mg_prep_bginput");
}
extern "C" int mg_nchw_to_nhwc(const float* in, float* out, int N, int C, int H, int W, int CP, const float* pmul,
                               void* stream) {
    if (!in || !out) return set_error(-1, "mg_nchw_to_nhwc: null pointer");
    nchw_to_nhwc_kernel<<<ew_grid((long long)N * H * W * CP), 256, 0, ST(stream)>>>(in, out, N, C, (long long)H * W, CP, pmul);
    return check_launch("mg_nchw_to_nhwc");
}
extern "C" int mg_nhwc_to_nchw(const float* in, float* out, int N, int C, int H, int W, int CP, void* stream) {
    if (!in || !out) return set_error(-1, "mg_nhwc_to_nchw: null pointer");
    nhwc_to_nchw_kernel<<<ew_grid((long long)N * C * H * W), 256, 0, ST(stream)>>>(in, out, N, C, (long long)H * W, CP);
    return check_launch("mg_nhwc_to_nchw");
}
extern "C" int mg_maxpool_mask(const float* in, float* out, float* tmp, int N, int H, int W, int k, int invert,
                               void* stream) {
    if (!in || !out || !tmp) return set_error(-1, "mg_maxpool_mask: null pointer");
    if (k % 2 != 1) return set_error(-2, "mg_maxpool_mask: k must be odd (got %d)", k);
    const long long total = (long long)N * H * W;
    maxfilt_kernel<<<ew_grid(total), 256, 0, ST(stream)>>>(in, tmp, N, H, W, k, 0, 0);
    count_launch();
    maxfilt_kernel<<<ew_grid(total), 256, 0, ST(stream)>>>(tmp, out, N, H, W, k, 1, invert);
    return check_launch("mg_maxpool_mask");
}
extern "C" int mg_avgpool3s2(const float* in, float* out, int N, int H, int W, int C, int OH, int OW, void* stream) {
    if (!in || !out) return set_error(-1, "mg_avgpool3s2: null pointer");
    if (C % 4 != 0) return set_error(-2, "mg_avgpool3s2: C%%4");
    avgpool3s2_kernel<<<ew_grid((long long)N * OH * OW * (C / 4)), 256, 0, ST(stream)>>>(in, out, N, H, W, C, OH, OW);
    return check_launch("mg_avgpool3s2");
}

extern "C" int mg_partial_mask(const float* mask, float* ratio, float* update, int N, int H, int W, int k, int stride,
                               int pad, void* stream) {
    if (!mask || !ratio || !update) return set_error(-1, "mg_partial_mask: null pointer");
    const int OH = (H + 2 * pad - k) / stride + 1, OW = (W + 2 * pad - k) / stride + 1;
    partial_mask_kernel<<<ew_grid((long long)N * OH * OW), 256, 0, ST(stream)>>>(mask, ratio, update, N, H, W, OH, OW, k,
                                                                               stride, pad);
    return check_launch("mg_partial_mask");
}
extern "C" int mg_masked_mean_bcast(const float* x, const float* mref, const float* mtag, float* out, int N, int h, int w,
                                    int C, int MH, int MW, void* stream) {
    if (!x || !mref || !mtag || !out) return set_error(-1, "mg_masked_mean_bcast: null pointer");
    if (MH % h != 0 || MW % w != 0) return set_error(-2, "mg_masked_mean_bcast: mask size must be a multiple of the map size");
    dim3 grid(cdiv(C, 32), N);
    masked_mean_bcast_kernel<<<grid, 256, 0, ST(stream)>>>(x, mref, mtag, out, N, h, w, C, MH, MW);
    return check_launch("mg_masked_mean_bcast");
}
extern "C" int mg_resize_bilinear(const float* in, float* out, int N, int H, int W, int C, int OH, int OW, void* stream) {
    if (!in || !out) return set_error(-1, "mg_resize_bilinear: null pointer");
    resize_bilinear_kernel<<<ew_grid((long long)N * OH * OW * C), 256, 0, ST(stream)>>>(in, out, N, H, W, C, OH, OW);
    return check_launch("mg_resize_bilinear");
}
extern "C" int mg_reflect_pad(const float* in, float* out, int N, int H, int W, int C, int pad, int round_tf32,
                              void* out_hi, void* out_lo, int out16_fmt, void* stream) {
    if (!in || (!out && !out_hi)) return set_error(-1, "mg_reflect_pad: null pointer");
    if (C % 4 != 0 || pad >= H || pad >= W) return set_error(-2, "mg_reflect_pad: C%%4==0 and pad < size required");
    reflect_pad_kernel<<<ew_grid((long long)N * (H + 2 * pad) * (W + 2 * pad) * (C / 4)), 256, 0, ST(stream)>>>(
        in, out, N, H, W, C, pad, round_tf32, (uint16_t*)out_hi, (uint16_t*)out_lo, out16_fmt);
    return check_launch("mg_reflect_pad");
}

// ------------------------------------------------------------------------------------ spectral norm (batched)
// torch SpectralNorm.compute_weight for every spectrally-normalised conv of a network in 3 launches
// (architecture.py:38-42, normalization.py:28-29): training -> v = normalize(W^T u), u = normalize(W v)
// in place; always sigma = u^T W v and inv_sigma = 1/sigma (consumed by mg_pack_weight).
namespace mg {
struct SnDesc {
    const float* w;   // [O][K]
    float* u;         // [O]
    float* v;         // [K]
    float* t;         // [K] workspace (zeroed by the caller)
    float* s;         // [O] workspace
    float* inv_sigma; // [1]
    int O, K;
};

__global__ void __launch_bounds__(128) sn_wtu_kernel(const SnDesc* __restrict__ descs, int row_splits) {
    const SnDesc d = descs[blockIdx.y];
    const int chunk = blockIdx.x / row_splits, split = blockIdx.x % row_splits;
    const int k = chunk * 128 + threadIdx.x;
    if (chunk * 128 >= d.K) return;
    const int rows_per = (d.O + row_splits - 1) / row_splits;
    const int r0 = split * rows_per, r1 = min(d.O, r0 + rows_per);
    if (k < d.K) {
        float acc = 0.f;
        for (int o = r0; o < r1; ++o) acc = fmaf(__ldg(d.w + (size_t)o * d.K + k), __ldg(d.u + o), acc);
        atomicAdd(d.t + k, acc);
    }
}
__global__ void __launch_bounds__(256) sn_wv_kernel(const SnDesc* __restrict__ descs, int training) {
    const SnDesc d = descs[blockIdx.y];
    const int o = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (o >= d.O) return;
    const int lane = threadIdx.x & 31;
    const float* vec = training ? d.t : d.v;
    const float* wr = d.w + (size_t)o * d.K;
    float acc = 0.f;
    for (int k = lane; k < d.K; k += 32) acc = fmaf(__ldg(wr + k), vec[k], acc);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) d.s[o] = acc;
}
__device__ float block_sum_256(float v, float* sh) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
    for (int i = 0; i < 8; ++i) r += sh[i];
    return r;
}
__global__ void __launch_bounds__(256) sn_finish_kernel(const SnDesc* __restrict__ descs, int training, float eps) {
    const SnDesc d = descs[blockIdx.x];
    __shared__ float sh[8];
    if (training) {
        float a = 0.f;
        for (int k = threadIdx.x; k < d.K; k += 256) a = fmaf(d.t[k], d.t[k], a);
        const float nt = fmaxf(sqrtf(block_sum_256(a, sh)), eps);
        float b = 0.f;
        for (int o = threadIdx.x; o < d.O; o += 256) { const float wv = d.s[o] / nt; b = fmaf(wv, wv, b); }
        const float n2 = block_sum_256(b, sh);
        const float nu = fmaxf(sqrtf(n2), eps);
        for (int k = threadIdx.x; k < d.K; k += 256) { d.v[k] = d.t[k] / nt; d.t[k] = 0.f; }
        for (int o = threadIdx.x; o < d.O; o += 256) d.u[o] = d.s[o] / nt / nu;
        if (threadIdx.x == 0) d.inv_sigma[0] = nu / n2;  // sigma = u.(Wv) = |Wv|^2 / nu
    } else {
        float a = 0.f;
        for (int o = threadIdx.x; o < d.O; o += 256) a = fmaf(d.u[o], d.s[o], a);
        const float sigma = block_sum_256(a, sh);
        if (threadIdx.x == 0) d.inv_sigma[0] = 1.f / sigma;
    }
}
}  // namespace mg

extern "C" int mg_spectral_norm_batched(const void* descs, int n_layers, int max_O, int max_K, int training, float eps,
                                        void* stream) {
    if (!descs || n_layers <= 0) return set_error(-1, "mg_spectral_norm_batched: bad arguments");
    const SnDesc* d = reinterpret_cast<const SnDesc*>(descs);
    if (training) {
        // one contribution per column (no split-K atomics): W^T u is then summed in a fixed order, so the power iteration is
        // bit-reproducible - every data-parallel rank derives IDENTICAL u, v, sigma from its identical weights (the reference's
        // replicas all read GPU 0's u, v).  Costs ~20 us per call against the 8-way split.
        const int splits = 1;
        dim3 g((unsigned)(cdiv(max_K, 128) * splits), (unsigned)n_layers);
        sn_wtu_kernel<<<g, 128, 0, ST(stream)>>>(d, splits);
        count_launch();
    }
    dim3 g2((unsigned)cdiv(max_O, 8), (unsigned)n_layers);
    sn_wv_kernel<<<g2, 256, 0, ST(stream)>>>(d, training);
    count_launch();
    sn_finish_kernel<<<n_layers, 256, 0, ST(stream)>>>(d, training, eps);
    return check_launch("mg_spectral_norm_batched");
}

// ------------------------------------------------------------------------------------ dgrad weight packing
// Data gradient of a conv = a stride-1 conv of dY with flipped, transposed (sub-)kernels.  For output
// parity (rh, rw) of a stride-s conv only taps kh = k0h + s*j contribute (see DESIGN.md "dgrad"):
//   out[ci][(th*Jw + tw)*O + co] = W[co][ci][k0h + s*(Jh-1-th)][k0w + s*(Jw-1-tw)] * inv_sigma
namespace mg {
__global__ void pack_weight_dgrad_kernel(const float* __restrict__ w, float* __restrict__ out, int O, int I, int KH, int KW,
                                         int s, int k0h, int Jh, int k0w, int Jw, const float* __restrict__ inv_sigma) {
    const long long total = (long long)I * Jh * Jw * O;
    const float sc = inv_sigma ? *inv_sigma : 1.f;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int co = idx % O;
        long long t = idx / O;
        const int tw = t % Jw; t /= Jw;
        const int th = t % Jh;
        const int ci = t / Jh;
        const int kh = k0h + s * (Jh - 1 - th), kw = k0w + s * (Jw - 1 - tw);
        out[idx] = rtf32(w[(((long long)co * I + ci) * KH + kh) * KW + kw] * sc);
    }
}
// packed [O][KH*KW*I] gradient -> OIHW (+= when accumulate)
__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, float* __restrict__ dw, int O, int I, int KH, int KW,
                                    int accumulate) {
    const long long total = (long long)O * I * KH * KW;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int kw = idx % KW;
        long long t = idx / KW;
        const int kh = t % KH; t /= KH;
        const int i = t % I;
        const int o = t / I;
        const float v = dwp[(size_t)o * KH * KW * I + (size_t)(kh * KW + kw) * I + i];
        dw[idx] = accumulate ? dw[idx] + v : v;
    }
}
}  // namespace mg

extern "C" int mg_pack_weight_dgrad(const float* w, float* out, int O, int I, int KH, int KW, int stride, int k0h, int Jh,
                                    int k0w, int Jw, const float* inv_sigma, void* stream) {
    if (!w || !out) return set_error(-1, "mg_pack_weight_dgrad: null pointer");
    if (k0h + stride * (Jh - 1) >= KH || k0w + stride * (Jw - 1) >= KW) return set_error(-2, "mg_pack_weight_dgrad: taps out of range");
    pack_weight_dgrad_kernel<<<ew_grid((long long)I * Jh * Jw * O), 256, 0, ST(stream)>>>(w, out, O, I, KH, KW, stride, k0h, Jh,
                                                                                         k0w, Jw, inv_sigma);
    return check_launch("mg_pack_weight_dgrad");
}
extern "C" int mg_unpack_wgrad(const float* dwp, float* dw_oihw, int O, int I, int KH, int KW, int accumulate, void* stream) {
    if (!dwp || !dw_oihw) return set_error(-1, "mg_unpack_wgrad: null pointer");
    unpack_wgrad_kernel<<<ew_grid((long long)O * I * KH * KW), 256, 0, ST(stream)>>>(dwp, dw_oihw, O, I, KH, KW, accumulate);
    return check_launch("mg_unpack_wgrad");
}

extern "C" int mg_pack_weight16(const float* w, void* out, int O, int I, int KH, int KW, const float* inv_sigma, int fmt,
                                int split, void* stream) {
    if (!w || !out) return set_error(-1, "mg_pack_weight16: null pointer");
    if (fmt < 1 || fmt > 2) return set_error(-2, "mg_pack_weight16: fmt must be 1 (fp16) or 2 (bf16)");
    pack_weight16_kernel<<<ew_grid((long long)O * I * KH * KW), 256, 0, ST(stream)>>>(w, (uint16_t*)out, O, I, KH, KW, inv_sigma,
                                                                                     fmt, split);
    return check_launch("mg_pack_weight16");
}
extern "C" int mg_pack_weight_gb16(const float* wg, const float* wb, void* out, int C, int I, int KH, int KW, int BN, int fmt,
                                   int split, void* stream) {
    if (!wg || !wb || !out) return set_error(-1, "mg_pack_weight_gb16: null pointer");
    if (BN % 64 != 0 || (2 * C) % BN != 0) return set_error(-2, "mg_pack_weight_gb16: bad BN %d for C %d", BN, C);
    pack_weight_gb16_kernel<<<ew_grid(2LL * C * I * KH * KW), 256, 0, ST(stream)>>>(wg, wb, (uint16_t*)out, C, I, KH, KW, BN, fmt, split);
    return check_launch("mg_pack_weight_gb16");
}

