// michigan_b200 — SPADE mlp_shared on tensor cores (normalization.py:92-96,110-111):
//     actv = ReLU(conv3x3(nearest_resize(segmap 4ch), W[128,4,3,3]) + b)
// The direct fp32 kernel (thin_conv_kernel) is FMA-bound (36 MACs x 128 channels per pixel).  Here the whole conv is ONE
// K = 128 GEMM per 128-pixel tile: builder warps gather the 3x3x4 patch of every pixel, split it into bf16 hi + lo and lay
// the row  [ hi(36) | lo(36) | hi(36) | 0(20) ]  down in the 128B-swizzled K-major operand layout; the resident weight
// operand is  [ W_hi | W_hi | W_lo | 0 ]  per output channel, so that the single accumulation
//     A_hi.W_hi + A_lo.W_hi + A_hi.W_lo      (~16 significand bits, same split as the other bf16x3 convs)
// comes out of 8 wgmma K steps (M 64 per warpgroup, N 128, K 16).  Warp roles: warps 0-7 = two consumer warpgroups (wgmma on
// pixel rows 0-63 / 64-127, accumulator -> smem tile -> bias/ReLU -> coalesced stores), warps 8-11 = operand builders (one
// pixel row each).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "mg_internal.h"
#include "mg_ptx.cuh"

namespace mg {

constexpr int kSegThreads = 32 * 12;
constexpr int kSegAccLd = 132;             // row pitch (floats) of the [128 x 128] accumulator tile
constexpr int kSegTileBytes = 2 * 16384;   // [128 rows x 128 K] bf16 as two K64 chunks of [128 x 128 B]

// MG_DBG & 16: clock64() totals of CTA 0 (read back with mg_debug_seg_prof)
__device__ unsigned long long g_seg_prof[16];

struct SegParams {
    const float* seg;     // [N, IH*R, IW*R, 4]
    const float* bias;    // [128]
    float* out;           // [N, OH, OW, 128] or null
    void* out_hi;         // 16-bit copy or null
    void* out_lo;
    int out16_fmt, round_out, act;
    int N, OH, OW, R;
    int tiles_w, tiles_h, num_tiles;
    int tma_store;   // 16-bit outputs leave through smem staging + TMA stores (out == null)
    int prof, dbg;   // dbg (MG_DBG bits, timing only): 1 no global stores, 2 no smem transposition
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(kSegThreads, 1)
seg_mlp_tc_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmHi,
                  const __grid_constant__ CUtensorMap tmLo, const SegParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* w_s = smem;                                    // resident weights
    uint8_t* a_s = smem + kSegTileBytes;                    // 2 operand buffers
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 3 * kSegTileBytes);
    uint64_t* a_full = bars;          // [2] 128 builder threads
    uint64_t* a_empty = bars + 2;     // [2] 8 consumer warps
    uint64_t* w_full = bars + 4;
    // fp32 [128][kSegAccLd] accumulator tile (1024-aligned); once a warp's columns are in registers its 8 KB share is also
    // that warp's TMA-store staging buffer
    float* acc_tile = reinterpret_cast<float*>(smem + 3 * kSegTileBytes + 1024);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmW);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&a_full[i], 128);
            mbar_init(&a_empty[i], 8);
        }
        mbar_init(w_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    const int tiles_per_img = p.tiles_w * p.tiles_h;

    if (warp < 8) {
        // ===================== consumers: wgmma (warpgroup wg = pixel rows 64*wg..), then the epilogue of 8 warps =====================
        if (warp == 0 && lane == 0) {
            mbar_arrive_expect_tx(w_full, kSegTileBytes);
            tma_load_2d(w_s, &tmW, w_full, 0, 0);
            tma_load_2d(w_s + 16384, &tmW, w_full, 64, 0);
        }
        mbar_wait(w_full, 0);
        const int wg = warp >> 2;
        const int quarter = warp & 3, half = warp >> 2, ew = warp;
        const int q = lane & 7, psub = lane >> 3;   // 8 lanes per pixel (32 channels), 4 pixels per pass
        // this warp's [32 px][64 ch] share of the accumulator tile, read transposed by the fp32 / register-store epilogue
        const float* scr = acc_tile + (size_t)(quarter * 32) * kSegAccLd + half * 64;
        float acc[64];
        int it = 0;
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
            const int s = it & 1;
            const uint32_t ph = (uint32_t)(it >> 1) & 1u;
            const int n = tile / tiles_per_img, m = tile - n * tiles_per_img;
            const int oh0 = (m / p.tiles_w) * 8, ow0 = (m % p.tiles_w) * 16;
            mbar_wait(&a_full[s], ph);
            const uint32_t a_addr = smem_u32(a_s + (size_t)s * kSegTileBytes) + (uint32_t)(wg * 64 * 128), w_addr = smem_u32(w_s);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const uint64_t da = wg_desc_sw128(a_addr + c * 16384, 1024), db = wg_desc_sw128(w_addr + c * 16384, 1024);
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_bf16_n128(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (c | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&a_empty[s]);
            // the previous tile's epilogue reads (and TMA stores out of the staging buffers) are done with the tile
            if (p.tma_store && it > 0) { if (lane == 0) tma_store_wait_read(); __syncwarp(); }
            bar_sync(1, 256);
            acc_store(acc_tile, kSegAccLd, acc, 128, wg * 64);
            bar_sync(1, 256);
            if (p.tma_store) {
                // 16-bit outputs only: lane = pixel row of a [32 px][64 ch] box (two image rows of the tile).  Each lane lays its
                // 128-byte row down in the SWIZZLE_128B pattern (16-byte chunk c at c ^ (row & 7): conflict-free per 8 lanes) and
                // one lane hands the 4 KB box to the TMA unit, which writes whole lines and clips the part outside the image.
                uint32_t v0[16], v1[16], v2[16], v3[16];
                const float* arow = acc_tile + (size_t)(quarter * 32 + lane) * kSegAccLd + half * 64;
                acc_ld16(arow, 0, v0); acc_ld16(arow, 16, v1); acc_ld16(arow, 32, v2); acc_ld16(arow, 48, v3);
                bar_sync(1, 256);
                uint8_t* st_hi = reinterpret_cast<uint8_t*>(acc_tile) + ew * 8192;
                uint8_t* st_lo = st_hi + 4096;
                const float* bsrc = p.bias + half * 64;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const uint32_t* v = (c >> 1) == 0 ? v0 : (c >> 1) == 1 ? v1 : (c >> 1) == 2 ? v2 : v3;
                    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bsrc + c * 8));
                    const float4 b1 = __ldg(reinterpret_cast<const float4*>(bsrc + c * 8 + 4));
                    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
                    float y[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        y[i] = __uint_as_float(v[(c & 1) * 8 + i]) + bb[i];
                        if (p.act == 1) y[i] = fmaxf(y[i], 0.f);
                        else if (p.act == 2) y[i] = y[i] > 0.f ? y[i] : 0.2f * y[i];
                        if (p.round_out) y[i] = round_tf32(y[i]);
                    }
                    uint32_t h[4], l[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float a = y[2 * i], b = y[2 * i + 1];
                        if (p.out16_fmt == 1) {
                            const __half2 h2 = __floats2half2_rn(fminf(fmaxf(a, -65504.f), 65504.f), fminf(fmaxf(b, -65504.f), 65504.f));
                            const float2 hf = __half22float2(h2);
                            const __half2 l2 = __floats2half2_rn(a - hf.x, b - hf.y);
                            h[i] = *reinterpret_cast<const uint32_t*>(&h2);
                            l[i] = *reinterpret_cast<const uint32_t*>(&l2);
                        } else {
                            const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
                            const float2 hf = __bfloat1622float2(h2);
                            h[i] = *reinterpret_cast<const uint32_t*>(&h2);
                            l[i] = pack_bf16x2(a - hf.x, b - hf.y);
                        }
                    }
                    const int off = lane * 128 + ((c ^ (lane & 7)) << 4);
                    *reinterpret_cast<uint4*>(st_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
                    if (p.out_lo) *reinterpret_cast<uint4*>(st_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0 && !(MG_DBGV(p) & 1)) {
                    tma_store_4d(&tmHi, st_hi, half * 64, ow0, oh0 + quarter * 2, n);
                    if (p.out_lo) tma_store_4d(&tmLo, st_lo, half * 64, ow0, oh0 + quarter * 2, n);
                    tma_store_commit();
                }
                continue;
            }
            // All 64 columns of this warp are read transposed so that every global store request is a full 128-byte line (the
            // SM->L2 write path is limited by requests, not bytes).  8 lanes serve one pixel: with a 16-bit
            // output each lane owns 8 consecutive channels (16 B -> 128 B per pixel and request); with an fp32 output it owns
            // channels q*4..q*4+3 and 32+q*4.. (two requests of 8 x 16 B = 128 B each).
            {
                const bool split = p.out != nullptr;                    // fp32 output present -> 4 + 4 channel ownership
                const int c0 = split ? q * 4 : q * 8, c1 = split ? 32 + q * 4 : q * 8 + 4;
                const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + half * 64 + c0));
                const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + half * 64 + c1));
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int r = quarter * 32 + j * 4 + psub;
                    const int oh = oh0 + (r >> 4), ow = ow0 + (r & 15);
                    const float4 t0v = *reinterpret_cast<const float4*>(scr + (j * 4 + psub) * kSegAccLd + c0);
                    const float4 t1v = *reinterpret_cast<const float4*>(scr + (j * 4 + psub) * kSegAccLd + c1);
                    if (oh >= p.OH || ow >= p.OW || ((MG_DBGV(p) & 1) && t0v.x != 12345.f)) continue;
                    float y[8] = {t0v.x + b0.x, t0v.y + b0.y, t0v.z + b0.z, t0v.w + b0.w, t1v.x + b1.x, t1v.y + b1.y, t1v.z + b1.z, t1v.w + b1.w};
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        if (p.act == 1) y[i] = fmaxf(y[i], 0.f);
                        else if (p.act == 2) y[i] = y[i] > 0.f ? y[i] : 0.2f * y[i];
                        if (p.round_out) y[i] = round_tf32(y[i]);
                    }
                    const size_t po = (((size_t)n * p.OH + oh) * p.OW + ow) * 128 + half * 64;
                    if (p.out) {
                        *reinterpret_cast<float4*>(p.out + po + c0) = make_float4(y[0], y[1], y[2], y[3]);
                        *reinterpret_cast<float4*>(p.out + po + c1) = make_float4(y[4], y[5], y[6], y[7]);
                    }
                    if (p.out_hi) {
                        uint32_t h[4], l[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float a = y[2 * i], b = y[2 * i + 1];
                            if (p.out16_fmt == 1) {
                                const __half2 h2 = __floats2half2_rn(fminf(fmaxf(a, -65504.f), 65504.f), fminf(fmaxf(b, -65504.f), 65504.f));
                                const float2 hf = __half22float2(h2);
                                const __half2 l2 = __floats2half2_rn(a - hf.x, b - hf.y);
                                h[i] = *reinterpret_cast<const uint32_t*>(&h2);
                                l[i] = *reinterpret_cast<const uint32_t*>(&l2);
                            } else {
                                const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
                                const float2 hf = __bfloat1622float2(h2);
                                h[i] = *reinterpret_cast<const uint32_t*>(&h2);
                                l[i] = pack_bf16x2(a - hf.x, b - hf.y);
                            }
                        }
                        uint16_t* ph16 = reinterpret_cast<uint16_t*>(p.out_hi) + po;
                        uint16_t* pl16 = p.out_lo ? reinterpret_cast<uint16_t*>(p.out_lo) + po : nullptr;
                        if (!split) {
                            *reinterpret_cast<uint4*>(ph16 + c0) = make_uint4(h[0], h[1], h[2], h[3]);
                            if (pl16) *reinterpret_cast<uint4*>(pl16 + c0) = make_uint4(l[0], l[1], l[2], l[3]);
                        } else {
                            *reinterpret_cast<uint2*>(ph16 + c0) = make_uint2(h[0], h[1]);
                            *reinterpret_cast<uint2*>(ph16 + c1) = make_uint2(h[2], h[3]);
                            if (pl16) {
                                *reinterpret_cast<uint2*>(pl16 + c0) = make_uint2(l[0], l[1]);
                                *reinterpret_cast<uint2*>(pl16 + c1) = make_uint2(l[2], l[3]);
                            }
                        }
                    }
                }
            }
        }
        if (p.tma_store && lane == 0) tma_store_wait_all();
    } else {
        // ===================== operand builders: thread = pixel row of the tile =====================
        const int r = threadIdx.x - 256;           // 0..127
        const int tw_l = r & 15, th_l = r >> 4;    // tile = 16 wide x 8 tall
        const int IH = p.OH, IW = p.OW;
        const size_t row_stride = (size_t)IW * p.R * 4, img_stride = (size_t)IH * p.R * row_stride;
        int it = 0;
        const bool prof = MG_PROFV(p) && blockIdx.x == 0 && r == 0;
        long long c_gather = 0, c_wait = 0, c_store = 0, t_begin = prof ? clock64() : 0;
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
            const int s = it & 1;
            const uint32_t ph = (uint32_t)(it >> 1) & 1u;
            const int n = tile / tiles_per_img, m = tile - n * tiles_per_img;
            const int oh = (m / p.tiles_w) * 8 + th_l, ow = (m % p.tiles_w) * 16 + tw_l;
            long long t0 = prof ? clock64() : 0;
            // gather the 3x3 neighbourhood (zero padding at the conv's resolution; nearest resize = index * R)
            uint2 hi[9], lo[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const int ih = oh + t / 3 - 1, iw = ow + t % 3 - 1;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (oh < IH && ih >= 0 && ih < IH && iw >= 0 && iw < IW)
                    v = __ldg(reinterpret_cast<const float4*>(p.seg + (size_t)n * img_stride + (size_t)ih * p.R * row_stride + (size_t)iw * p.R * 4));
                const __nv_bfloat162 h01 = __floats2bfloat162_rn(v.x, v.y), h23 = __floats2bfloat162_rn(v.z, v.w);
                const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
                hi[t] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
                lo[t] = make_uint2(pack_bf16x2(v.x - f01.x, v.y - f01.y), pack_bf16x2(v.z - f23.x, v.w - f23.y));
            }
            if (prof) { const long long t1 = clock64(); c_gather += t1 - t0; t0 = t1; }
            mbar_wait(&a_empty[s], ph ^ 1);
            if (prof) { const long long t1 = clock64(); c_wait += t1 - t0; t0 = t1; }
            uint8_t* base = a_s + (size_t)s * kSegTileBytes + (size_t)r * 128;
            // K order: 8-byte groups g = 0..31: hi taps 0..8 | lo taps 0..8 | hi taps 0..8 | zeros
            auto group = [&](int g) -> uint2 {
                if (g < 9) return hi[g];
                if (g < 18) return lo[g - 9];
                if (g < 27) return hi[g - 18];
                return make_uint2(0u, 0u);
            };
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const uint2 g0 = group(2 * u), g1 = group(2 * u + 1);
                const int c = u >> 3, j = u & 7;
                *reinterpret_cast<uint4*>(base + c * 16384 + ((j ^ (r & 7)) << 4)) = make_uint4(g0.x, g0.y, g1.x, g1.y);
            }
            fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core (async proxy)
            mbar_arrive(&a_full[s]);
            if (prof) c_store += clock64() - t0;
        }
        if (prof) {
            g_seg_prof[3] = (unsigned long long)(clock64() - t_begin); g_seg_prof[4] = (unsigned long long)c_gather;
            g_seg_prof[5] = (unsigned long long)c_wait; g_seg_prof[6] = (unsigned long long)c_store;
        }
    }
}

// w [128][Cin<=4][3][3] fp32 -> bf16 [128][128]: k = part*36 + tap*4 + ci, parts (W_hi, W_hi, W_lo), zero tail.
__global__ void pack_weight_seg_tc_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cin) {
    const int co = blockIdx.x, k = threadIdx.x;   // 128 x 128
    float val = 0.f;
    int part = 3;
    if (k < 108) {
        part = k / 36;
        const int r = k - part * 36, tap = r >> 2, ci = r & 3;
        if (ci < Cin) val = w[((size_t)co * Cin + ci) * 9 + tap];
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(val);
    const __nv_bfloat16 lo = __float2bfloat16_rn(val - __bfloat162float(hi));
    out[(size_t)co * 128 + k] = part == 2 ? lo : (part < 2 ? hi : __float2bfloat16_rn(0.f));
}

}  // namespace mg

using namespace mg;

// Debug: [3] builder total, [4] gather, [5] wait operand-empty, [6] store+fence (CTA 0, probe build with MG_DBG & 16).
extern "C" int mg_debug_seg_prof(unsigned long long* host16) {
    if (!host16) return set_error(-1, "mg_debug_seg_prof: null pointer");
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(host16, g_seg_prof, 16 * sizeof(unsigned long long));
    if (e != cudaSuccess) return set_error((int)e, "mg_debug_seg_prof: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int mg_pack_weight_seg_tc(const float* w_oihw, void* wpack, int O, int I, void* stream_) {
    if (!w_oihw || !wpack) return set_error(-1, "mg_pack_weight_seg_tc: null pointer");
    if (O != 128 || I < 1 || I > 4) return set_error(-2, "mg_pack_weight_seg_tc: needs O = 128, I <= 4 (got %d, %d)", O, I);
    pack_weight_seg_tc_kernel<<<128, 128, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(w_oihw, reinterpret_cast<__nv_bfloat16*>(wpack), I);
    return check_launch("mg_pack_weight_seg_tc");
}

// Same contract as mg_conv_thin for the SPADE mlp_shared geometry (CinP 4, 3x3, stride 1, pad 1 zero, Cout 128);
// a->w is the bf16 operand produced by mg_pack_weight_seg_tc.
extern "C" int mg_conv_seg_tc(const mg_thin_args* a, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->in || !a->w || !a->bias || (!a->out && !a->out_hi)) return set_error(-1, "mg_conv_seg_tc: null pointer");
    if (a->CinP != 4 || a->KH != 3 || a->KW != 3 || a->stride != 1 || a->pad != 1 || a->pad_mode != 0 || a->Cout != 128 || a->pscale || a->pmul)
        return set_error(-2, "mg_conv_seg_tc: only the SPADE mlp_shared geometry (4 -> 128, 3x3 s1 p1) is supported");
    if (a->OH != a->H || a->OW != a->W) return set_error(-3, "mg_conv_seg_tc: output size must equal the (virtual) input size");
    if (a->out_hi && (a->out16_fmt < 1 || a->out16_fmt > 2)) return set_error(-4, "mg_conv_seg_tc: out16_fmt must be 1 or 2");
    SegParams p;
    memset(&p, 0, sizeof(p));
    p.seg = a->in; p.bias = a->bias; p.out = a->out; p.out_hi = a->out_hi; p.out_lo = a->out_lo; p.out16_fmt = a->out16_fmt;
    p.round_out = a->round_out; p.act = a->act;
    p.N = a->N; p.OH = a->OH; p.OW = a->OW; p.R = a->seg_resize > 0 ? a->seg_resize : 1;
    p.tiles_w = (a->OW + 15) / 16; p.tiles_h = (a->OH + 7) / 8; p.num_tiles = p.tiles_w * p.tiles_h * a->N;
#ifdef MG_PROBES
    p.prof = probe_bits() & 16;
    p.dbg = probe_bits() & 3;
#endif
    CUtensorMap tmW;
    {
        cuuint64_t dims[2] = {128, 128};
        cuuint64_t strides[1] = {128 * 2};
        cuuint32_t box[2] = {64, 128};
        cuuint32_t es[2] = {1, 1};
        int rc = encode_tensor_map(&tmW, (void*)a->w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    CUtensorMap tmHi = tmW, tmLo = tmW;
    p.tma_store = (tune(TK_SEG_TMA) && !a->out && a->out_hi) ? 1 : 0;
    if (p.tma_store) {
        // [N][OH][OW][128] 16-bit, box = 64 channels x 16 x 2 pixels = one epilogue warp's share of a tile
        cuuint64_t dims[4] = {128, (cuuint64_t)a->OW, (cuuint64_t)a->OH, (cuuint64_t)a->N};
        cuuint64_t strides[3] = {128 * 2, (cuuint64_t)a->OW * 256, (cuuint64_t)a->OW * a->OH * 256};
        cuuint32_t box[4] = {64, 16, 2, 1};
        cuuint32_t es[4] = {1, 1, 1, 1};
        const CUtensorMapDataType dt = a->out16_fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
        int rc = encode_tensor_map(&tmHi, a->out_hi, dt, 4, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
        if (!rc && a->out_lo) rc = encode_tensor_map(&tmLo, a->out_lo, dt, 4, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const size_t smem_bytes = 1024 + 3 * kSegTileBytes + 1024 + 128 * kSegAccLd * 4;
    static thread_local int attr_dev = -1;
    int dev = 0; cudaGetDevice(&dev);
    if (attr_dev != dev) {
        cudaError_t e = cudaFuncSetAttribute(seg_mlp_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) return set_error((int)e, "mg_conv_seg_tc attr: %s", cudaGetErrorString(e));
        attr_dev = dev;
    }
    int grid = num_sms();
    if (grid > p.num_tiles) grid = p.num_tiles;
    seg_mlp_tc_kernel<<<grid, kSegThreads, smem_bytes, stream>>>(tmW, tmHi, tmLo, p);
    return check_launch("mg_conv_seg_tc");
}
