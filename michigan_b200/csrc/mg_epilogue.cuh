// michigan_b200 — shared pieces of the implicit-GEMM convolution kernels: the parameter block and the transposed,
// coalesced epilogue (accumulator tile in shared memory -> bias / residual / blend / SPADE modulation -> global memory).
// Used by mg_igemm.cu (per-tap operand loads) and mg_conv3x3.cu (halo patches, M-tile groups).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "mg_ptx.cuh"
#include "mg_internal.h"

namespace mg {

constexpr int kNumEpiWarps = 8;
// warps 0..7: two consumer warpgroups (wgmma on rows 0-63 / 64-127 of the 128-pixel tile, then the epilogue), warp 8: TMA producer
constexpr int kThreads = kNumEpiWarps * 32 + 32;  // 288
constexpr int kMaxAccCols = 128;                  // accumulator columns per tile: 64 fp32 registers per consumer thread
constexpr int kABytes = 128 * 128;                // 128 pixels x 32 fp32
constexpr int kMaxStages = 8;
constexpr int kMaxASlots = 4;

struct IgemmParams {
    int N, OH, OW, Cout;
    int Cin, KH, KW, stride, pad_h, pad_w;
    int os, ooh, oow, OHF, OWF, accumulate;
    int TW, TH, TN, tiles_w, tiles_h, tiles_n;
    int BN, n_tiles, num_tiles, kchunks, stages;
    int epi, act, round_out;
    int a_fmt, parts, kelem;      // operand format: 0 tf32 (32 ch / 128 B row), 1 fp16, 2 bf16 (64 ch / row); parts 1 or 3
    float* out;                   // fp32 output (may be null when only 16-bit copies are wanted)
    void* out_hi;                 // optional 16-bit copy of the output (operand of the next tensor-core conv)
    void* out_lo;                 // optional 16-bit residual: cvt(y - float(hi))
    int out16_fmt;                // 1 fp16, 2 bf16
    const float* bias;
    const float* res;
    int res_shift, RH, RW;
    const float* pscale;
    const float* pmul;
    const float* bf;
    const float* hair;
    const float* back;
    int mask_stride, MH, MW;
    const float* x;
    int x_shift, XH, XW;
    const float* nscale;
    const float* nshift;
    const float* gbias1;
    const float* bbias;
    float* aux;   // SPADE: optional [N,OH,OW,Cout] copy of (1 + gamma) for the backward pass
    int epi_impl, epi_cw16, epi_off;   // 1 = transposed/coalesced epilogue (default), 0 = row-per-lane; scratch offset in smem
    int acc_off, acc_ld;               // smem accumulator tile: byte offset, row pitch in floats (acc_cols + 4: conflict-free rows)
    // halo mode (3x3, stride 1, pad 1): one [PW x (TH+2)] input patch per K chunk serves all 9 taps
    int halo, PW, patch_bytes, patch_tx, a_slots, b_slots, b_slot_bytes, acc_cols, merged, n_items, bar_off;
    int dbg;   // what-if probes (env MG_DBG; 1..8 give WRONG results): 1 no B loads after the first tile, 2 no A loads, 4 no epilogue work, 8 no epilogue global traffic (32 no 16-bit stores only, 64 no x loads only), 16 cycle profile
};

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == 1) return fmaxf(v, 0.f);
    if (act == 2) return v > 0.f ? v : 0.2f * v;
    if (act == 3) return tanhf(v);
    return v;
}


// One accumulator tile (128 pixels x BN columns, fp32 [128][ld] in shared memory) through the epilogue, executed by the 8
// consumer warps together (warp -> row quarter `quarter` = warp & 3 and column half `half`).  Each lane reads one
// accumulator ROW (pixel); the raw accumulators of a CW-channel chunk are dumped to a warp-private smem scratch `scr`
// (32 x (CW + 4) floats) and read back transposed, so that in the arithmetic and in every global access a group of 4/8
// lanes covers one pixel's contiguous channels (full 64/128 B segments) instead of 32 lanes touching 32 different lines.
// SPEC selects a compile-time specialisation of the (instruction-bound) epilogue:
//   0 generic (everything decided at run time)
//   1 SPADE + LeakyReLU -> bf16 hi/lo operand only      2 SPADE + no activation -> bf16 hi/lo operand only
// CW: channels per epilogue chunk (16 or 32), compile time so that the per-chunk register arrays are sized exactly.
template <int SPEC, int CW>
__device__ __forceinline__ void epilogue_tile(const IgemmParams& p, float* scr, const float* acc, int nt, int tw, int th, int tn,
                                              int quarter, int half, int lane) {
    constexpr bool kS = SPEC == 1 || SPEC == 2;
    const bool spade = kS ? true : (p.epi == 1);
    const int act = SPEC == 1 ? 2 : (SPEC == 2 ? 0 : p.act);
    const bool has_out = kS ? false : (p.out != nullptr);
    const bool has_hi = kS ? true : (p.out_hi != nullptr);
    const bool has_lo = kS ? true : (p.out_lo != nullptr);
    const int fmt16 = kS ? 2 : p.out16_fmt;
    const bool has_aux = kS ? false : (p.aux != nullptr);
    const bool do_round = kS ? false : (p.round_out != 0);
    const int span = spade ? (p.BN >> 2) : (p.BN >> 1);   // channels this warp owns per tile
    constexpr int cw = CW;
    constexpr int rs = cw + 4;
    constexpr int lpp = cw >> 2, ppp = 32 / lpp, passes = lpp;   // lanes per pixel, pixels per pass, passes per chunk
    const int q = lane % lpp, psub = lane / lpp;
    const int twl = 31 - __clz(p.TW), thl = 31 - __clz(p.TH);
    const int ch_tile = p.BN >> 1;
    // per-tile pixel bookkeeping for the (up to 8) pixels this lane serves in the transposed domain
    uint32_t pixo[passes], srco[passes];
    uint32_t vmask = 0;
#pragma unroll
    for (int j = 0; j < passes; ++j) {
        pixo[j] = srco[j] = 0;
        const int r = quarter * 32 + j * ppp + psub;
        const int ow = tw * p.TW + (r & (p.TW - 1));
        const int oh = th * p.TH + ((r >> twl) & (p.TH - 1));
        const int n = tn * p.TN + (r >> (twl + thl));
        if (ow >= p.OW || oh >= p.OH || n >= p.N) continue;
        vmask |= 1u << j;
        pixo[j] = (uint32_t)(((size_t)n * p.OHF + (size_t)oh * p.os + p.ooh) * p.OWF + (size_t)ow * p.os + p.oow);
        if (spade) srco[j] = (uint32_t)(((size_t)n * p.XH + (oh >> p.x_shift)) * p.XW + (ow >> p.x_shift));
        else if (p.res) srco[j] = (uint32_t)(((size_t)n * p.RH + (oh >> p.res_shift)) * p.RW + (ow >> p.res_shift));
    }
    const float* t_row = acc + (size_t)(quarter * 32 + lane) * p.acc_ld;
    for (int cb = 0; cb < span; cb += cw) {
        if (MG_DBGV(p) & 4) break;
        const int col = half * span + cb;          // first column of this chunk (gamma part for SPADE)
        float4 av[passes], bv[passes], pre[passes];
        const int cch = (spade ? nt * ch_tile : nt * p.BN) + col + q * 4;
        uint32_t g0[16], g1[16], b0[16], b1[16];
        // registers (row per lane) -> scratch -> registers (transposed: lanes cover contiguous channels)
        auto transpose = [&](const uint32_t (&v0)[16], const uint32_t (&v1)[16], float4 (&dst)[passes], bool add) {
            float4* d = reinterpret_cast<float4*>(scr + lane * rs);
#pragma unroll
            for (int i = 0; i < 4; ++i)
                d[i] = make_float4(__uint_as_float(v0[4 * i]), __uint_as_float(v0[4 * i + 1]), __uint_as_float(v0[4 * i + 2]),
                                   __uint_as_float(v0[4 * i + 3]));
            if (cw == 32) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    d[4 + i] = make_float4(__uint_as_float(v1[4 * i]), __uint_as_float(v1[4 * i + 1]), __uint_as_float(v1[4 * i + 2]),
                                           __uint_as_float(v1[4 * i + 3]));
            }
            __syncwarp();
#pragma unroll
            for (int j = 0; j < passes; ++j) {
                const float4 t = *reinterpret_cast<const float4*>(scr + (j * ppp + psub) * rs + q * 4);
                if (add) { dst[j].x += t.x; dst[j].y += t.y; dst[j].z += t.z; dst[j].w += t.w; }
                else dst[j] = t;
            }
            __syncwarp();
        };
        auto load_chunk = [&](int colbase, float4 (&dst)[passes], bool add) {
            uint32_t v0[16], v1[16];
            acc_ld16(t_row, colbase, v0);
            if (cw == 32) acc_ld16(t_row, colbase + 16, v1);
            transpose(v0, v1, dst, add);
        };
        acc_ld16(t_row, col, g0);
        if (cw == 32) acc_ld16(t_row, col + 16, g1);
        if (spade) {
            acc_ld16(t_row, col + ch_tile, b0);
            if (cw == 32) acc_ld16(t_row, col + ch_tile + 16, b1);
        }
        const bool ch_ok = cch < p.Cout;
        transpose(g0, g1, av, false);
        // Per-pixel side loads (SPADE: the tensor being normalised; else the residual): issued as soon as the first
        // transposition has freed its registers, so their L2 latency overlaps the second one.
        const float* side = spade ? p.x : p.res;
        if (side != nullptr && ch_ok && !(MG_DBGV(p) & (8 | 64))) {
#pragma unroll
            for (int j = 0; j < passes; ++j)
                if ((vmask >> j) & 1u) pre[j] = __ldg(reinterpret_cast<const float4*>(side + (size_t)srco[j] * p.Cout + cch));
        }
        if (p.merged) load_chunk(col + p.BN, av, true);   // split precision, merged N: + A_hi * W_lo columns
        if (spade) transpose(b0, b1, bv, false);
        float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f), sc4 = bias4, sh4 = bias4, g14 = bias4, bb4 = bias4;
        if (ch_ok) {
            if (spade) {
                sc4 = __ldg(reinterpret_cast<const float4*>(p.nscale + cch));
                sh4 = __ldg(reinterpret_cast<const float4*>(p.nshift + cch));
                g14 = __ldg(reinterpret_cast<const float4*>(p.gbias1 + cch));
                bb4 = __ldg(reinterpret_cast<const float4*>(p.bbias + cch));
            } else if (p.bias) {
                bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + cch));
            }
        }
        if (spade) {
            // fold gamma into the normalised input right away (frees `pre` before beta is fetched):
            // av <- (x * rstd + shift) * (1 + gamma)
#pragma unroll
            for (int j = 0; j < passes; ++j) {
                if (!((vmask >> j) & 1u) || !ch_ok) continue;
                const float4 xv = (MG_DBGV(p) & (8 | 64)) ? sc4 : pre[j];
                const float4 gs = make_float4(g14.x + av[j].x, g14.y + av[j].y, g14.z + av[j].z, g14.w + av[j].w);
                if (has_aux) *reinterpret_cast<float4*>(p.aux + (size_t)pixo[j] * p.Cout + cch) = gs;
                av[j] = make_float4(fmaf(xv.x, sc4.x, sh4.x) * gs.x, fmaf(xv.y, sc4.y, sh4.y) * gs.y,
                                    fmaf(xv.z, sc4.z, sh4.z) * gs.z, fmaf(xv.w, sc4.w, sh4.w) * gs.w);
            }
            if (p.merged) load_chunk(col + ch_tile + p.BN, bv, true);
        }
        if (!ch_ok) continue;
#pragma unroll
        for (int j = 0; j < passes; ++j) {
            if (!((vmask >> j) & 1u)) continue;
            const size_t pix = pixo[j];
            float y[4];
            if (spade) {
                y[0] = av[j].x + (bb4.x + bv[j].x); y[1] = av[j].y + (bb4.y + bv[j].y);
                y[2] = av[j].z + (bb4.z + bv[j].z); y[3] = av[j].w + (bb4.w + bv[j].w);
#pragma unroll
                for (int i = 0; i < 4; ++i) y[i] = apply_act(y[i], act);
            } else {
                const float ps = p.pscale ? __ldg(p.pscale + pix) : 1.f;
                y[0] = fmaf(av[j].x, ps, bias4.x); y[1] = fmaf(av[j].y, ps, bias4.y);
                y[2] = fmaf(av[j].z, ps, bias4.z); y[3] = fmaf(av[j].w, ps, bias4.w);
                if (p.res) {
                    const float4 rv = pre[j];
                    y[0] += rv.x; y[1] += rv.y; y[2] += rv.z; y[3] += rv.w;
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) y[i] = apply_act(y[i], act);
                if (p.bf) {
                    // full-resolution mask coordinates of this output pixel (blend epilogue only)
                    const int rr = quarter * 32 + j * ppp + psub;
                    const size_t mp = ((size_t)(tn * p.TN + (rr >> (twl + thl))) * p.MH +
                                       (size_t)(th * p.TH + ((rr >> twl) & (p.TH - 1))) * p.mask_stride) * p.MW +
                                      (size_t)(tw * p.TW + (rr & (p.TW - 1))) * p.mask_stride;
                    const float om_hair = 1.f - __ldg(p.hair + mp), om_back = 1.f - __ldg(p.back + mp);
                    const float4 bfv = __ldg(reinterpret_cast<const float4*>(p.bf + pix * p.Cout + cch));
                    y[0] = bfv.x * om_hair + y[0] * om_back; y[1] = bfv.y * om_hair + y[1] * om_back;
                    y[2] = bfv.z * om_hair + y[2] * om_back; y[3] = bfv.w * om_hair + y[3] * om_back;
                }
                if (p.pmul) {
                    const float pm = __ldg(p.pmul + pix);
#pragma unroll
                    for (int i = 0; i < 4; ++i) y[i] *= pm;
                }
            }
            if (do_round) {
#pragma unroll
                for (int i = 0; i < 4; ++i) y[i] = round_tf32(y[i]);
            }
            if (has_out) {
                float4* op = reinterpret_cast<float4*>(p.out + pix * p.Cout + cch);
                if (p.accumulate) {
                    const float4 o = *op;
                    y[0] += o.x; y[1] += o.y; y[2] += o.z; y[3] += o.w;
                }
                *op = make_float4(y[0], y[1], y[2], y[3]);
            }
            if (has_hi && !((MG_DBGV(p) & (8 | 32)) && y[0] != 12345.f)) {
                uint32_t hi[2], lo[2];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const float a = y[2 * i], b = y[2 * i + 1];
                    if (fmt16 == 1) {
                        const __half2 h2 = __floats2half2_rn(fminf(fmaxf(a, -65504.f), 65504.f), fminf(fmaxf(b, -65504.f), 65504.f));
                        const float2 hf = __half22float2(h2);
                        const __half2 l2 = __floats2half2_rn(a - hf.x, b - hf.y);
                        hi[i] = *reinterpret_cast<const uint32_t*>(&h2);
                        lo[i] = *reinterpret_cast<const uint32_t*>(&l2);
                    } else {
                        const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
                        const float2 hf = __bfloat1622float2(h2);
                        const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - hf.x, b - hf.y);
                        hi[i] = *reinterpret_cast<const uint32_t*>(&h2);
                        lo[i] = *reinterpret_cast<const uint32_t*>(&l2);
                    }
                }
                const size_t eo = pix * p.Cout + cch;
                *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(p.out_hi) + eo) = make_uint2(hi[0], hi[1]);
                if (has_lo) *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(p.out_lo) + eo) = make_uint2(lo[0], lo[1]);
            }
        }
    }
}

}  // namespace mg
