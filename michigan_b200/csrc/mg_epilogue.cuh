// michigan_b200 — shared pieces of the implicit-GEMM convolution kernels: the parameter block and the transposed,
// coalesced epilogue (accumulator tile in shared memory -> bias / residual / blend / SPADE modulation -> global memory).
// Used by mg_igemm.cu (per-tap operand loads) and mg_conv3x3.cu (halo patches, M-tile groups).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <type_traits>
#include "mg_ptx.cuh"
#include "mg_internal.h"

namespace mg {

constexpr int kNumEpiWarps = 8;
// warps 0..7: two consumer warpgroups (wgmma on rows 0-63 / 64-127 of the 128-pixel tile, then the epilogue);
// warps 8..11: the producer warpgroup, in which one thread issues the TMA loads.  A whole warpgroup for the producer lets it
// hand registers back with setmaxnreg: 40 x 128 + 232 x 256 = 64,512 of the SM's 65,536.
constexpr int kThreads = kNumEpiWarps * 32 + 128;  // 384
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(kProducerRegs * 128 + kConsumerRegs * kNumEpiWarps * 32 <= 65536, "register split exceeds the SM's file");
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
    int dbg;   // what-if probes (env MG_DBG; 1..8 give WRONG results): 1 no B loads after the first tile, 2 no A loads, 4 no epilogue work, 8 no epilogue global traffic (32 no 16-bit stores only, 64 no x loads only)
};

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == 1) return fmaxf(v, 0.f);
    if (act == 2) return v > 0.f ? v : 0.2f * v;
    if (act == 3) return tanhf(v);
    return v;
}

// ---------------------------------------------------------------------------------------------- per-element arithmetic
// epilogue_tile and epilogue_frag hold an element in different threads but must give it the same bits: both call these.
// Every product that a later add could absorb is rounded explicitly (__fmul_rn, or fmaf where the fusion is wanted):
// whether the compiler contracts a plain a * b + c depends on the code around it, which differs between the two epilogues.
// SPADE, first half: gs = 1 + gamma (gbias1 folds the 1 and gamma's bias); returns (x * rstd + shift) * (1 + gamma).
__device__ __forceinline__ float epi_spade_mod(float x, float sc, float sh, float g1, float gacc, float& gs) {
    gs = g1 + gacc;
    return __fmul_rn(fmaf(x, sc, sh), gs);
}
// SPADE, second half: + beta (with its bias), activation.
__device__ __forceinline__ float epi_spade_out(float m, float bb, float bacc, int act) { return apply_act(m + (bb + bacc), act); }
// Plain conv: per-pixel scale, bias, residual, activation.
__device__ __forceinline__ float epi_plain(float a, float ps, float bias, bool has_res, float r, int act) {
    float y = fmaf(a, ps, bias);
    if (has_res) y += r;
    return apply_act(y, act);
}
// Background blend: bf where the hair / background masks say so.
__device__ __forceinline__ float epi_blend(float y, float bfv, float om_hair, float om_back) {
    return fmaf(om_hair, bfv, __fmul_rn(om_back, y));
}
// Per-pixel output multiplier (pmul).
__device__ __forceinline__ float epi_pmul(float y, float pm) { return __fmul_rn(y, pm); }
// Two consecutive channels -> packed 16-bit hi and lo = cvt(y - float(hi)); fp16 clamps hi to its finite range.
__device__ __forceinline__ void epi_split16(float a, float b, int fmt16, uint32_t& hi, uint32_t& lo) {
    if (fmt16 == 1) {
        const __half2 h2 = __floats2half2_rn(fminf(fmaxf(a, -65504.f), 65504.f), fminf(fmaxf(b, -65504.f), 65504.f));
        const float2 hf = __half22float2(h2);
        const __half2 l2 = __floats2half2_rn(a - hf.x, b - hf.y);
        hi = *reinterpret_cast<const uint32_t*>(&h2);
        lo = *reinterpret_cast<const uint32_t*>(&l2);
    } else {
        const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
        const float2 hf = __bfloat1622float2(h2);
        const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - hf.x, b - hf.y);
        hi = *reinterpret_cast<const uint32_t*>(&h2);
        lo = *reinterpret_cast<const uint32_t*>(&l2);
    }
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
                float4 gs, m;
                m.x = epi_spade_mod(xv.x, sc4.x, sh4.x, g14.x, av[j].x, gs.x);
                m.y = epi_spade_mod(xv.y, sc4.y, sh4.y, g14.y, av[j].y, gs.y);
                m.z = epi_spade_mod(xv.z, sc4.z, sh4.z, g14.z, av[j].z, gs.z);
                m.w = epi_spade_mod(xv.w, sc4.w, sh4.w, g14.w, av[j].w, gs.w);
                if (has_aux) *reinterpret_cast<float4*>(p.aux + (size_t)pixo[j] * p.Cout + cch) = gs;
                av[j] = m;
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
                y[0] = epi_spade_out(av[j].x, bb4.x, bv[j].x, act); y[1] = epi_spade_out(av[j].y, bb4.y, bv[j].y, act);
                y[2] = epi_spade_out(av[j].z, bb4.z, bv[j].z, act); y[3] = epi_spade_out(av[j].w, bb4.w, bv[j].w, act);
            } else {
                const float ps = p.pscale ? __ldg(p.pscale + pix) : 1.f;
                const bool has_res = p.res != nullptr;
                const float4 rv = has_res ? pre[j] : bias4;
                y[0] = epi_plain(av[j].x, ps, bias4.x, has_res, rv.x, act); y[1] = epi_plain(av[j].y, ps, bias4.y, has_res, rv.y, act);
                y[2] = epi_plain(av[j].z, ps, bias4.z, has_res, rv.z, act); y[3] = epi_plain(av[j].w, ps, bias4.w, has_res, rv.w, act);
                if (p.bf) {
                    // full-resolution mask coordinates of this output pixel (blend epilogue only)
                    const int rr = quarter * 32 + j * ppp + psub;
                    const size_t mp = ((size_t)(tn * p.TN + (rr >> (twl + thl))) * p.MH +
                                       (size_t)(th * p.TH + ((rr >> twl) & (p.TH - 1))) * p.mask_stride) * p.MW +
                                      (size_t)(tw * p.TW + (rr & (p.TW - 1))) * p.mask_stride;
                    const float om_hair = 1.f - __ldg(p.hair + mp), om_back = 1.f - __ldg(p.back + mp);
                    const float4 bfv = __ldg(reinterpret_cast<const float4*>(p.bf + pix * p.Cout + cch));
                    y[0] = epi_blend(y[0], bfv.x, om_hair, om_back); y[1] = epi_blend(y[1], bfv.y, om_hair, om_back);
                    y[2] = epi_blend(y[2], bfv.z, om_hair, om_back); y[3] = epi_blend(y[3], bfv.w, om_hair, om_back);
                }
                if (p.pmul) {
                    const float pm = __ldg(p.pmul + pix);
#pragma unroll
                    for (int i = 0; i < 4; ++i) y[i] = epi_pmul(y[i], pm);
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
                for (int i = 0; i < 2; ++i) epi_split16(y[2 * i], y[2 * i + 1], fmt16, hi[i], lo[i]);
                const size_t eo = pix * p.Cout + cch;
                *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(p.out_hi) + eo) = make_uint2(hi[0], hi[1]);
                if (has_lo) *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(p.out_lo) + eo) = make_uint2(lo[0], lo[1]);
            }
        }
    }
}

// The rest of the epilogue of one output pair (channels ch, ch + 1 of pixel pix): rounding, fp32 store (or accumulation), 16-bit
// hi/lo copies.
template <int SPEC>
__device__ __forceinline__ void epi_store_pair(const IgemmParams& p, size_t pix, int ch, float y0, float y1) {
    constexpr bool kS = SPEC == 1 || SPEC == 2;
    if (!kS && p.round_out != 0) { y0 = round_tf32(y0); y1 = round_tf32(y1); }
    const size_t eo = pix * p.Cout + ch;
    if (!kS && p.out != nullptr) {
        float2* op = reinterpret_cast<float2*>(p.out + eo);
        if (p.accumulate) {
            const float2 o = *op;
            y0 += o.x; y1 += o.y;
        }
        *op = make_float2(y0, y1);
    }
    if ((kS || p.out_hi != nullptr) && !((MG_DBGV(p) & (8 | 32)) && y0 != 12345.f)) {
        uint32_t hi, lo;
        epi_split16(y0, y1, kS ? 2 : p.out16_fmt, hi, lo);
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out_hi) + eo) = hi;
        if (kS || p.out_lo != nullptr) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out_lo) + eo) = lo;
    }
}

// The same for the SPADE epilogue of epilogue_frag: rounding, fp32 store (or accumulation) when `store`, and the packed 16-bit
// hi/lo words, which epi_store16_quad writes.
template <int SPEC>
__device__ __forceinline__ void epi_finish_pair(const IgemmParams& p, size_t pix, int ch, bool store, float y0, float y1, uint32_t& hi,
                                                uint32_t& lo) {
    constexpr bool kS = SPEC == 1 || SPEC == 2;
    if (!kS && p.round_out != 0) { y0 = round_tf32(y0); y1 = round_tf32(y1); }
    if (!kS && p.out != nullptr && store) {
        float2* op = reinterpret_cast<float2*>(p.out + pix * p.Cout + ch);
        if (p.accumulate) {
            const float2 o = *op;
            y0 += o.x; y1 += o.y;
        }
        *op = make_float2(y0, y1);
    }
    if (kS || p.out_hi != nullptr) epi_split16(y0, y1, kS ? 2 : p.out16_fmt, hi, lo);
}

// 4 x 4 transposition of 32-bit words across the lanes of a quad (two butterfly steps): lane q's w[i] becomes lane i's w[q].
// Every lane of the warp must take part.
__device__ __forceinline__ void quad_transpose(uint32_t (&w)[4], int lane) {
    const bool b1 = (lane & 2) != 0, b0 = (lane & 1) != 0;
    uint32_t s0 = b1 ? w[0] : w[2], s1 = b1 ? w[1] : w[3];
    s0 = __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 = __shfl_xor_sync(0xffffffffu, s1, 2);
    if (b1) { w[0] = s0; w[1] = s1; } else { w[2] = s0; w[3] = s1; }
    s0 = b0 ? w[0] : w[1];
    s1 = b0 ? w[2] : w[3];
    s0 = __shfl_xor_sync(0xffffffffu, s0, 1);
    s1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    if (b0) { w[0] = s0; w[2] = s1; } else { w[1] = s0; w[3] = s1; }
}

// The 16-bit copies of four 8-channel blocks of one pixel: hi[i] / lo[i] hold this lane's pair 2 (lane & 3) of block i, whose
// first channel is cb + 8 i.  After a quad transposition lane q holds all four pairs of block q and writes them with one 16-byte
// store, so a quad writes 64 contiguous bytes (whole 32-byte sectors) instead of four lanes x 4 bytes per block.  Every lane
// of the warp must call it; `store` masks the pixel.  Cout is a multiple of 32 (every N tile is full), so a block is either
// wholly inside the output or wholly outside, and pix * Cout * 2 bytes is 16-byte aligned.
template <int SPEC>
__device__ __forceinline__ void epi_store16_quad(const IgemmParams& p, size_t pix, int cb, bool store, uint32_t (&hi)[4],
                                                 uint32_t (&lo)[4], int lane) {
    constexpr bool kS = SPEC == 1 || SPEC == 2;
    if (!kS && p.out_hi == nullptr) return;
    const bool has_lo = kS || p.out_lo != nullptr;
    quad_transpose(hi, lane);
    if (has_lo) quad_transpose(lo, lane);
    const int ch = cb + 8 * (lane & 3);
    if (!store || ch >= p.Cout || ((MG_DBGV(p) & (8 | 32)) && hi[0] != 12345u)) return;
    const size_t eo = pix * p.Cout + ch;
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out_hi) + eo) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    if (has_lo) *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out_lo) + eo) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// The two finished M tiles of a conv3x3_group_kernel group (TW = 8, TH = 16, TN = 1) straight from the wgmma accumulators:
// no shared-memory tile, no transposition, no barrier.  Thread (warpgroup wg, warp quarter = warp & 3, lane) holds in acc_t
// rows 64 wg + 16 quarter + lane/4 + 8h (h = 0, 1) of M tile t, i.e. pixel (ow = 8 (tw0 + t) + lane/4, oh = 16 th + 8 wg +
// 2 quarter + h), and in register 4j + 2h + e the accumulator column 8j + 2 (lane & 3) + e.  So every thread owns 4 pixels and
// a fixed set of channel pairs, and what the epilogue combines is in the same thread: SPADE's gamma and beta (columns c and
// c + BN/2) and the two halves of merged split precision (c and c + BN).  The per-pixel side inputs of a tile (SPADE x or the
// residual, blend maps, pscale / pmul) are loaded before its arithmetic; the per-channel parameters are read through L1 (both
// tiles' accumulators and x leave no registers to keep them for the whole group).  SPADE's 16-bit copies are transposed
// across each quad and written 16 bytes per lane (epi_store16_quad).  The plain epilogue keeps 4-byte 16-bit stores: the
// transposition's words do not fit next to its side inputs at merged BN = 64 without spills.
// Same arithmetic as epilogue_tile (the epi_* helpers), so every element gets the same bits.
template <int SPEC, int BN, bool MERGED, int R>
__device__ __forceinline__ void epilogue_frag(const IgemmParams& p, const float (&acc0)[R], const float (&acc1)[R], int nt, int tw0,
                                              int th, int tn, int wg, int quarter, int lane) {
    constexpr bool kS = SPEC == 1 || SPEC == 2;
    constexpr int kLo = BN / 8;   // register-group offset of accumulator column c + BN (merged split precision)
    static_assert(R == (MERGED ? BN : BN / 2), "accumulator registers: 64 x N per warpgroup is N / 2 per thread");
    const int act = SPEC == 1 ? 2 : (SPEC == 2 ? 0 : p.act);
    if (MG_DBGV(p) & 4) return;
    const int c0 = 2 * (lane & 3);
    // the thread's pixels: [tile][h]
    size_t pix[2][2], src[2][2];
    bool ok[2][2];
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int ow = (tw0 + t) * 8 + (lane >> 2), oh = th * 16 + 8 * wg + 2 * quarter + h, n = tn;
            ok[t][h] = ow < p.OW && oh < p.OH;
            pix[t][h] = ((size_t)n * p.OHF + (size_t)oh + p.ooh) * p.OWF + (size_t)ow + p.oow;
            if (kS || p.epi == 1) src[t][h] = ((size_t)n * p.XH + (oh >> p.x_shift)) * p.XW + (ow >> p.x_shift);
            else src[t][h] = ((size_t)n * p.RH + (oh >> p.res_shift)) * p.RW + (ow >> p.res_shift);
        }
    const bool side_ok = !(MG_DBGV(p) & (8 | 64));

    if constexpr (BN % 64 == 0) {
        if (kS || p.epi == 1) {
            // ---- SPADE: out = act((x * rstd + shift) * (1 + gamma) + beta), gamma | beta packed [BN/2 | BN/2]
            constexpr int J = BN / 16, kBeta = BN / 16;
            const int ch0 = nt * (BN / 2) + c0;   // channel of accumulator column 8j + c0: ch0 + 8j
            const bool has_aux = !kS && p.aux != nullptr;
            float2 xv[2][2][J];
            auto load_x = [&](auto tc) {
                constexpr int t = decltype(tc)::value;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int j = 0; j < J; ++j)
                        xv[t][h][j] = ok[t][h] && side_ok && ch0 + 8 * j < p.Cout
                                          ? __ldg(reinterpret_cast<const float2*>(p.x + src[t][h] * p.Cout + ch0 + 8 * j))
                                          : make_float2(0.f, 0.f);
            };
            // blocks of four column groups j (32 channels): the 16-bit words of a block leave through epi_store16_quad, so the
            // arithmetic runs for masked pixels too (their loads and stores are skipped) and every lane reaches the shuffles
            auto block = [&](const float (&acc)[R], auto tc, int k) {
                constexpr int t = decltype(tc)::value;
                {
                    uint32_t hi[2][4], lo[2][4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int j = 4 * k + i, ch = ch0 + 8 * j;
                        const bool cok = ch < p.Cout;
                        const float2 z = make_float2(0.f, 0.f);
                        const float2 sc = cok ? __ldg(reinterpret_cast<const float2*>(p.nscale + ch)) : z;
                        const float2 sh = cok ? __ldg(reinterpret_cast<const float2*>(p.nshift + ch)) : z;
                        const float2 g1 = cok ? __ldg(reinterpret_cast<const float2*>(p.gbias1 + ch)) : z;
                        const float2 bb = cok ? __ldg(reinterpret_cast<const float2*>(p.bbias + ch)) : z;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const bool st = ok[t][h] && cok;
                            const float2 x = side_ok ? xv[t][h][j] : sc;
                            float g[2], b[2], gs[2], y[2];
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                g[e] = acc[4 * j + 2 * h + e];
                                b[e] = acc[4 * (j + kBeta) + 2 * h + e];
                                if (MERGED) {
                                    g[e] += acc[4 * (j + kLo) + 2 * h + e];
                                    b[e] += acc[4 * (j + kBeta + kLo) + 2 * h + e];
                                }
                            }
                            y[0] = epi_spade_out(epi_spade_mod(x.x, sc.x, sh.x, g1.x, g[0], gs[0]), bb.x, b[0], act);
                            y[1] = epi_spade_out(epi_spade_mod(x.y, sc.y, sh.y, g1.y, g[1], gs[1]), bb.y, b[1], act);
                            if (has_aux && st) *reinterpret_cast<float2*>(p.aux + pix[t][h] * p.Cout + ch) = make_float2(gs[0], gs[1]);
                            epi_finish_pair<SPEC>(p, pix[t][h], ch, st, y[0], y[1], hi[h][i], lo[h][i]);
                        }
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) epi_store16_quad<SPEC>(p, pix[t][h], ch0 - c0 + 32 * k, ok[t][h], hi[h], lo[h], lane);
                }
            };
            // SPEC 1/2 fetch tile 1's x once tile 0's first block has freed its registers, so that its latency overlaps the
            // rest of tile 0; the generic variant fetches it after tile 0
            using T0 = std::integral_constant<int, 0>;
            using T1 = std::integral_constant<int, 1>;
            load_x(T0{});
            block(acc0, T0{}, 0);
            if constexpr (kS) load_x(T1{});
#pragma unroll
            for (int k = 1; k < J / 4; ++k) block(acc0, T0{}, k);
            if constexpr (!kS) load_x(T1{});
#pragma unroll
            for (int k = 0; k < J / 4; ++k) block(acc1, T1{}, k);
            return;
        }
    }
    if constexpr (!kS) {
        // ---- plain conv: out = pmul * blend(act(acc * pscale + bias + res))
        constexpr int J = BN / 8;
        const int ch0 = nt * BN + c0;
        const bool has_res = p.res != nullptr, has_bf = p.bf != nullptr;
        // one pixel row (tile t, row h) at a time: its side loads first, then its arithmetic
        auto row = [&](const float (&acc)[R], auto tc, auto hc) {
            constexpr int t = decltype(tc)::value, h = decltype(hc)::value;
            if (!ok[t][h]) return;
            float2 rv[J], bfv[J];
            const float ps = p.pscale ? __ldg(p.pscale + pix[t][h]) : 1.f;
            const float pm = p.pmul ? __ldg(p.pmul + pix[t][h]) : 1.f;
            float om_hair = 0.f, om_back = 0.f;
            if (has_bf) {
                const int ow = (tw0 + t) * 8 + (lane >> 2), oh = th * 16 + 8 * wg + 2 * quarter + h;
                const size_t mp = ((size_t)tn * p.MH + (size_t)oh * p.mask_stride) * p.MW + (size_t)ow * p.mask_stride;
                om_hair = 1.f - __ldg(p.hair + mp);
                om_back = 1.f - __ldg(p.back + mp);
            }
#pragma unroll
            for (int j = 0; j < J; ++j) {
                const bool cok = ch0 + 8 * j < p.Cout;
                rv[j] = cok && has_res && side_ok ? __ldg(reinterpret_cast<const float2*>(p.res + src[t][h] * p.Cout + ch0 + 8 * j))
                                                  : make_float2(0.f, 0.f);
                bfv[j] = cok && has_bf ? __ldg(reinterpret_cast<const float2*>(p.bf + pix[t][h] * p.Cout + ch0 + 8 * j))
                                       : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int j = 0; j < J; ++j) {
                const int ch = ch0 + 8 * j;
                if (ch >= p.Cout) continue;
                const float2 bias = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + ch)) : make_float2(0.f, 0.f);
                float a[2], y[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    a[e] = acc[4 * j + 2 * h + e];
                    if (MERGED) a[e] += acc[4 * (j + kLo) + 2 * h + e];
                }
                y[0] = epi_plain(a[0], ps, bias.x, has_res, rv[j].x, act);
                y[1] = epi_plain(a[1], ps, bias.y, has_res, rv[j].y, act);
                if (has_bf) {
                    y[0] = epi_blend(y[0], bfv[j].x, om_hair, om_back);
                    y[1] = epi_blend(y[1], bfv[j].y, om_hair, om_back);
                }
                if (p.pmul) { y[0] = epi_pmul(y[0], pm); y[1] = epi_pmul(y[1], pm); }
                epi_store_pair<SPEC>(p, pix[t][h], ch, y[0], y[1]);
            }
        };
        using I0 = std::integral_constant<int, 0>;
        using I1 = std::integral_constant<int, 1>;
        row(acc0, I0{}, I0{});
        row(acc0, I0{}, I1{});
        row(acc1, I1{}, I0{});
        row(acc1, I1{}, I1{});
    }
}

// ------------------------------------------------------------------------------------------------ kernel variants
// The tensor-core conv kernels are compiled per (operand format FMT, BN, MERGED, SPEC, CW) so that every wgmma of their
// mainloops has a compile-time shape and type.  MERGED = merged split precision: A_hi x [W_hi ; W_lo] at N = 2*BN plus
// A_lo x W_hi at N = BN into a 2*BN-column accumulator.  Only the combinations igemm_launch can select are instantiated:
//   merged      16-bit operands and 2*BN <= 128
//   SPEC 1, 2   SPADE epilogue, so BN % 64 == 0
//   CW 32       needs 32 | the channels a warp owns per tile (BN/2, SPADE BN/4): BN >= 64, SPADE specialisations BN = 128
template <int FMT, int BN, bool MERGED, int SPEC, int CW>
constexpr bool conv_variant_exists() {
    return (!MERGED || (FMT != 0 && 2 * BN <= kMaxAccCols)) && (SPEC == 0 || BN % 64 == 0) &&
           (CW == 16 || (SPEC == 0 ? BN >= 64 : BN == 128));
}

// Calls L::run<FMT, BN, MERGED, SPEC, CW>() for run-time values; run() returns an error status for a combination that
// conv_variant_exists rejects, and so does this function for values outside the template domain.
template <int FMT, int BN, bool MERGED, int SPEC, class L>
int dispatch_cw(const L& l, int cw) {
    if (cw == 16) return l.template run<FMT, BN, MERGED, SPEC, 16>();
    if (cw == 32) return l.template run<FMT, BN, MERGED, SPEC, 32>();
    return set_error(-14, "conv kernel: no variant for epilogue chunk width %d", cw);
}
template <int FMT, int BN, bool MERGED, class L>
int dispatch_spec(const L& l, int spec, int cw) {
    if (spec == 0) return dispatch_cw<FMT, BN, MERGED, 0>(l, cw);
    if (spec == 1) return dispatch_cw<FMT, BN, MERGED, 1>(l, cw);
    if (spec == 2) return dispatch_cw<FMT, BN, MERGED, 2>(l, cw);
    return set_error(-14, "conv kernel: no variant for epilogue specialisation %d", spec);
}
template <int FMT, int BN, class L>
int dispatch_merged(const L& l, bool merged, int spec, int cw) {
    return merged ? dispatch_spec<FMT, BN, true>(l, spec, cw) : dispatch_spec<FMT, BN, false>(l, spec, cw);
}
template <int FMT, class L>
int dispatch_bn(const L& l, int bn, bool merged, int spec, int cw) {
    if (bn == 32) return dispatch_merged<FMT, 32>(l, merged, spec, cw);
    if (bn == 64) return dispatch_merged<FMT, 64>(l, merged, spec, cw);
    if (bn == 128) return dispatch_merged<FMT, 128>(l, merged, spec, cw);
    return set_error(-14, "conv kernel: no variant for BN %d", bn);
}
template <class L>
int dispatch_conv_variant(const L& l, int fmt, int bn, bool merged, int spec, int cw) {
    if (fmt == 0) return dispatch_bn<0>(l, bn, merged, spec, cw);
    if (fmt == 1) return dispatch_bn<1>(l, bn, merged, spec, cw);
    if (fmt == 2) return dispatch_bn<2>(l, bn, merged, spec, cw);
    return set_error(-14, "conv kernel: no variant for operand format %d", fmt);
}

// Launches `kernel` with the whole opt-in shared memory, setting the attribute once per device and variant.
template <class K, class... Args>
int launch_conv_kernel(K* kernel, int& attr_dev, int grid, size_t smem_bytes, cudaStream_t stream, const Args&... args) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_dev != dev) {
        const cudaError_t e = cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return set_error((int)e, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        attr_dev = dev;
    }
    kernel<<<grid, kThreads, smem_bytes, stream>>>(args...);
    count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error((int)e, "conv kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

}  // namespace mg
