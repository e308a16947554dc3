// michigan_b200 — im2col-free implicit-GEMM convolution on wgmma (sm_90a).
//
//   D[pixels(128) x BN] += sum_{tap, cin-chunk} A_tap[pixels x 32] * W[BN x 32]^T
//
// * activations NHWC; one TMA 4-D box per (tap, 32-channel chunk): the box start is shifted by the
//   tap offset and TMA's out-of-bounds zero fill implements the conv zero padding; strided convs
//   use the tensor map's elementStrides (traversal stride) so no im2col / space-to-depth copy exists;
// * weights pre-packed tap-major [CoutG][KH*KW*Cin] and loaded by a 2-D TMA box;
// * both operands land in 128B-swizzled K-major smem tiles that wgmma reads directly; the fp32
//   accumulator lives in the registers of two consumer warpgroups (rows 0-63 / 64-127 of the tile)
//   and goes through a shared-memory tile to the epilogue those same 8 warps run; the producer
//   keeps filling the stage ring meanwhile;
// * warp roles: warps 0..7 = wgmma consumers + epilogue (232 registers each), warps 8..11 = producer
//   warpgroup (40 registers; one thread issues the TMA loads);
// * mainloop: compile-time wgmma shape and format, one wgmma group kept in flight (wait_group 1),
//   a stage released once the wait that retires its MMAs has passed;
// * persistent CTAs (<= 1 per SM), static round-robin tile schedule with the N-tile index fastest
//   so CTAs running concurrently share activation tiles through L2.
//
// Epilogues: bias/activation/residual/background-blend, and the fused SPADE modulation
// (normalization.py:116 + architecture.py:84-85 of the reference).
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <type_traits>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "mg_ptx.cuh"
#include "mg_internal.h"
#include "mg_epilogue.cuh"

namespace mg {

// 16 consecutive channels -> 16-bit hi (and optional lo = cvt(y - hi)) copies, 32 B each.
__device__ __forceinline__ void store16(const IgemmParams& p, const float (&y)[16], size_t elem_off) {
    uint32_t hi[8], lo[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float a = y[2 * i], b = y[2 * i + 1];
        if (p.out16_fmt == 1) {
            const __half ha = __float2half_rn(fminf(fmaxf(a, -65504.f), 65504.f));
            const __half hb = __float2half_rn(fminf(fmaxf(b, -65504.f), 65504.f));
            hi[i] = (uint32_t)__half_as_ushort(ha) | ((uint32_t)__half_as_ushort(hb) << 16);
            const __half la = __float2half_rn(a - __half2float(ha)), lb = __float2half_rn(b - __half2float(hb));
            lo[i] = (uint32_t)__half_as_ushort(la) | ((uint32_t)__half_as_ushort(lb) << 16);
        } else {
            const __nv_bfloat16 ha = __float2bfloat16_rn(a), hb = __float2bfloat16_rn(b);
            hi[i] = (uint32_t)__bfloat16_as_ushort(ha) | ((uint32_t)__bfloat16_as_ushort(hb) << 16);
            const __nv_bfloat16 la = __float2bfloat16_rn(a - __bfloat162float(ha)), lb = __float2bfloat16_rn(b - __bfloat162float(hb));
            lo[i] = (uint32_t)__bfloat16_as_ushort(la) | ((uint32_t)__bfloat16_as_ushort(lb) << 16);
        }
    }
    uint4* ph = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out_hi) + elem_off);
    ph[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    ph[1] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
    if (p.out_lo) {
        uint4* pl = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out_lo) + elem_off);
        pl[0] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        pl[1] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
    }
}

// FMT (operand format), BN and MERGED fix the shape and type of every wgmma (see conv_variant_exists in mg_epilogue.cuh).
// SPEC selects a compile-time specialisation of the (instruction-bound) epilogue:
//   0 generic (everything decided at run time)
//   1 SPADE + LeakyReLU -> bf16 hi/lo operand only      2 SPADE + no activation -> bf16 hi/lo operand only
// CW: channels per epilogue chunk (16 or 32), compile time so that the per-chunk register arrays are sized exactly.
template <int FMT, int BN, bool MERGED, int SPEC, int CW>
__global__ void __launch_bounds__(kThreads, 1)
igemm_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                  const __grid_constant__ CUtensorMap tmB, const IgemmParams p) {
    constexpr int kAcc = MERGED ? 2 * BN : BN;   // accumulator columns
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // 1024-align the operand ring (SWIZZLE_128B atoms are 1024 B).
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int stage_bytes = kABytes + p.acc_cols * 128;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.bar_off);
    uint64_t* full_bar = bars;                        // halo mode: the weight (B) ring
    uint64_t* empty_bar = bars + kMaxStages;
    uint64_t* afull_bar = bars + 2 * kMaxStages;      // halo mode: the patch (A) ring, <= kMaxASlots slots
    uint64_t* aempty_bar = afull_bar + kMaxASlots;
    float* acc_tile = reinterpret_cast<float*>(smem + p.acc_off);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == kNumEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmA2);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < (p.halo ? p.b_slots : p.stages); ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kNumEpiWarps);
        }
        for (int s = 0; s < p.a_slots; ++s) {
            mbar_init(&afull_bar[s], 1);
            mbar_init(&aempty_bar[s], kNumEpiWarps);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const int ksteps = p.KH * p.KW * p.parts * p.kchunks;
    const int m_tiles_per_img = p.tiles_w * p.tiles_h;

    if (warp >= kNumEpiWarps) {
        // The producer warpgroup hands its registers to the consumers; one thread of it issues every TMA load.
        setmaxnreg_dec<kProducerRegs>();
        if (warp != kNumEpiWarps || lane != 0) return;
    }
    if (warp == kNumEpiWarps && p.halo) {
        // ===================== TMA producer, halo mode (one thread) =====================
        // Two rings: A = input patches (one per K chunk [x hi/lo part], reused by all 9 taps), B = weights
        // (one slot per tap).  A patches are prefetched up to a_slots-1 items ahead of the weight stream.
        {
            const int parts2 = p.merged ? 2 : 1;
            const int bparts = p.merged ? 2 : 1;
            uint8_t* a_ring = smem;
            uint8_t* b_ring = smem + (size_t)p.a_slots * p.patch_bytes;
            int bs = 0, as_ = 0;
            uint32_t bph = 0, aphs = 0;
            long long a_issued = 0, b_item = 0;
            int tileA = blockIdx.x, itA = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                const int nt = tile % p.n_tiles;
                for (int it = 0; it < p.n_items; ++it, ++b_item) {
                    const int kc = it / parts2, part = it - kc * parts2;
                    for (int tap = 0; tap < 9; ++tap) {
                        while (tileA < p.num_tiles && a_issued < b_item + p.a_slots) {
                            const bool must = a_issued <= b_item;
                            if (!must && !mbar_test_wait(&aempty_bar[as_], aphs ^ 1)) break;
                            if (must) mbar_wait_report(&aempty_bar[as_], aphs ^ 1);
                            const int mA = tileA / p.n_tiles;
                            const int twA = mA % p.tiles_w, thA = (mA / p.tiles_w) % p.tiles_h, tnA = mA / m_tiles_per_img;
                            const int kcA = itA / parts2, partA = itA - kcA * parts2;
                            mbar_arrive_expect_tx(&afull_bar[as_], (uint32_t)p.patch_tx);
                            tma_load_4d(a_ring + (size_t)as_ * p.patch_bytes, partA ? &tmA2 : &tmA, &afull_bar[as_], kcA * p.kelem,
                                        twA * p.TW - 1, thA * p.TH - 1, tnA);
                            if (++as_ == p.a_slots) { as_ = 0; aphs ^= 1; }
                            if (++itA == p.n_items) { itA = 0; tileA += gridDim.x; }
                            ++a_issued;
                        }
                        mbar_wait_report(&empty_bar[bs], bph ^ 1);
                        uint8_t* sb = b_ring + (size_t)bs * p.b_slot_bytes;
                        const int kofs = tap * bparts * p.Cin + kc * p.kelem;
                        if (p.merged && part == 0) {
                            // A_hi x [W_hi ; W_lo]: both weight parts side by side -> one N = 2*BN MMA
                            mbar_arrive_expect_tx(&full_bar[bs], (uint32_t)(2 * p.BN * 128));
                            tma_load_2d(sb, &tmB, &full_bar[bs], kofs, nt * p.BN);
                            tma_load_2d(sb + p.BN * 128, &tmB, &full_bar[bs], kofs + p.Cin, nt * p.BN);
                        } else {
                            mbar_arrive_expect_tx(&full_bar[bs], (uint32_t)(p.BN * 128));
                            tma_load_2d(sb, &tmB, &full_bar[bs], kofs, nt * p.BN);
                        }
                        if (++bs == p.b_slots) { bs = 0; bph ^= 1; }
                    }
                }
            }
        }
    } else if (warp == kNumEpiWarps) {
        // ===================== TMA producer (one thread) =====================
        {
            int st = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                const bool ldA = !(MG_DBGV(p) & 2) || tile == (int)blockIdx.x, ldB = !(MG_DBGV(p) & 1) || tile == (int)blockIdx.x;
                const int nt = tile % p.n_tiles;
                const int m = tile / p.n_tiles;
                const int tw = m % p.tiles_w;
                const int th = (m / p.tiles_w) % p.tiles_h;
                const int tn = m / m_tiles_per_img;
                const int iw0 = tw * p.TW * p.stride - p.pad_w;
                const int ih0 = th * p.TH * p.stride - p.pad_h;
                const int n0 = tn * p.TN;
                const int bparts = p.parts >= 2 ? 2 : 1;   // weight operand holds (hi) or (hi, lo) per tap
                for (int tap = 0; tap < p.KH * p.KW; ++tap) {
                    const int kh = tap / p.KW, kw = tap - kh * p.KW;
                    for (int part = 0; part < p.parts; ++part) {
                        // split precision, 3 passes: A_hi*W_hi + A_lo*W_hi + A_hi*W_lo
                        // merged (2 passes): A_hi x [W_hi ; W_lo] (N = 2*BN) + A_lo x W_hi (N = BN)
                        const CUtensorMap* ta = part == 1 ? &tmA2 : &tmA;
                        const int bsel = part == 2 ? 1 : 0;
                        const bool both = p.merged && part == 0;
                        for (int kc = 0; kc < p.kchunks; ++kc) {
                            mbar_wait_report(&empty_bar[st], ph ^ 1);
                            uint8_t* sa = smem + (size_t)st * stage_bytes;
                            const uint32_t txs = (ldA ? kABytes : 0) + (ldB ? p.BN * 128 * (both ? 2 : 1) : 0);
                            if (txs == 0) { mbar_arrive(&full_bar[st]); }
                            else mbar_arrive_expect_tx(&full_bar[st], txs);
                            if (ldA) tma_load_4d(sa, ta, &full_bar[st], kc * p.kelem, iw0 + kw, ih0 + kh, n0);
                            const int kofs = (tap * bparts + bsel) * p.Cin + kc * p.kelem;
                            if (ldB) {
                                tma_load_2d(sa + kABytes, &tmB, &full_bar[st], kofs, nt * p.BN);
                                if (both) tma_load_2d(sa + kABytes + p.BN * 128, &tmB, &full_bar[st], kofs + p.Cin, nt * p.BN);
                            }
                            if (++st == p.stages) { st = 0; ph ^= 1; }
                        }
                    }
                }
            }
        }
    } else {
        // ===================== consumers: warpgroup wg multiplies rows 64*wg.. of the tile, then all 8 warps run the epilogue
        setmaxnreg_inc<kConsumerRegs>();
        const int wg = warp >> 2;
        const int quarter = warp & 3;           // rows 32*quarter.. of the accumulator tile in the epilogue
        const int half = warp >> 2;             // column half handled by this warp in the epilogue
        float* scr = reinterpret_cast<float*>(smem + p.epi_off) + warp * (32 * (CW + 4));
        float acc[kAcc / 2];
        int st = 0, bs = 0, as_ = 0;
        uint32_t ph = 0, bph = 0, aphs = 0;
        const uint32_t ring = smem_u32(smem);
        // Pipelined mainloop: one wgmma group stays in flight.  After a step commits, wait_group 1 retires the step before
        // it, and only then is that step's B slot (classic mode: its whole stage) released; an A patch (halo mode) is
        // released by the wait that retires its last step.  held_*: slots whose release waits for that retirement.
        int held_b = -1, held_a = -1;
        auto release_held = [&]() {
            __syncwarp();
            if (lane == 0) {   // this warp's reads of the slots are done
                if (held_b >= 0) mbar_arrive(&empty_bar[held_b]);
                if (held_a >= 0) mbar_arrive(&aempty_bar[held_a]);
            }
            held_b = held_a = -1;
        };
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            const int nt = tile % p.n_tiles;
            const int m = tile / p.n_tiles;
            const int tw = m % p.tiles_w;
            const int th = (m / p.tiles_w) % p.tiles_h;
            const int tn = m / m_tiles_per_img;
            if (p.halo) {
                constexpr int parts2 = MERGED ? 2 : 1;
                const uint32_t b_ring = ring + (uint32_t)(p.a_slots * p.patch_bytes);
                for (int it = 0; it < p.n_items; ++it) {
                    mbar_wait(&afull_bar[as_], aphs);
                    // rows 64.. of the tile are its pixel rows 8.., eight patch rows of PW pixels further on
                    const uint32_t a_base = ring + (uint32_t)(as_ * p.patch_bytes) + (uint32_t)(wg * 8 * p.PW * 128);
                    // the nine taps of one item at MMA width N
                    auto item = [&](auto n_cols) {
                        constexpr int N = decltype(n_cols)::value;
                        for (int tap = 0; tap < 9; ++tap) {
                            const int kh = tap / 3, kw = tap - kh * 3;
                            mbar_wait(&full_bar[bs], bph);
                            // tap (kh, kw) = the same patch read from row kh*PW + kw on; 8-pixel row groups are PW rows apart
                            const uint32_t a_tap = a_base + (uint32_t)((kh * p.PW + kw) * 128);
                            const uint64_t db = wg_desc_sw128(b_ring + (uint32_t)(bs * p.b_slot_bytes), 1024);
                            wgmma_fence();
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                const uint64_t da = wg_desc_sw128(a_tap + (uint32_t)(k * 32), (uint32_t)(p.PW * 128));
                                wgmma_step<FMT, N>(acc, da, db + (uint64_t)(2 * k), (it | tap | k) != 0 ? 1u : 0u);
                            }
                            wgmma_commit();
                            wgmma_wait<1>();
                            release_held();
                            held_b = bs;
                            if (++bs == p.b_slots) { bs = 0; bph ^= 1; }
                        }
                    };
                    // merged split precision: items alternate between A_hi x [W_hi ; W_lo] (N = 2*BN) and A_lo x W_hi (N = BN)
                    if (MERGED && it % parts2 == 1) item(std::integral_constant<int, BN>{});
                    else item(std::integral_constant<int, kAcc>{});
                    held_a = as_;
                    if (++as_ == p.a_slots) { as_ = 0; aphs ^= 1; }
                }
            } else {
                // one run = the K chunks of one (tap, part) at MMA width N
                auto run = [&](int ks0, auto n_cols) {
                    constexpr int N = decltype(n_cols)::value;
                    for (int ks = ks0; ks < ks0 + p.kchunks; ++ks) {
                        mbar_wait(&full_bar[st], ph);
                        const uint32_t sa = ring + (uint32_t)(st * stage_bytes);
                        const uint64_t da = wg_desc_sw128(sa + (uint32_t)(wg * 64 * 128), 1024);
                        const uint64_t db = wg_desc_sw128(sa + kABytes, 1024);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k)   // advance 32 B inside the 128 B swizzle row: +2 in 16 B units
                            wgmma_step<FMT, N>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (ks | k) != 0 ? 1u : 0u);
                        wgmma_commit();
                        wgmma_wait<1>();
                        release_held();
                        held_b = st;
                        if (++st == p.stages) { st = 0; ph ^= 1; }
                    }
                };
                // merged split precision: runs alternate between N = 2*BN and N = BN
                for (int ks0 = 0; ks0 < ksteps; ks0 += p.kchunks) {
                    if (MERGED && ((ks0 / p.kchunks) & 1)) run(ks0, std::integral_constant<int, BN>{});
                    else run(ks0, std::integral_constant<int, kAcc>{});
                }
            }
            wgmma_wait<0>();
            wgmma_fence_operand(acc);
            release_held();
            bar_sync(1, kNumEpiWarps * 32);     // the previous tile's epilogue is done with the accumulator tile
            acc_store(acc_tile, p.acc_ld, acc, kAcc, wg * 64);
            bar_sync(1, kNumEpiWarps * 32);
            if (p.epi_impl == 1) {
                epilogue_tile<SPEC, CW>(p, scr, acc_tile, nt, tw, th, tn, quarter, half, lane);
                continue;
            }
            // ===================== row-per-lane reference epilogue =====================
            const int r = quarter * 32 + lane;      // accumulator row == pixel within tile
            const int wl = r % p.TW;
            const int hl = (r / p.TW) % p.TH;
            const int nl = r / (p.TW * p.TH);
            const int ow = tw * p.TW + wl;
            const int oh = th * p.TH + hl;
            const int n = tn * p.TN + nl;
            const bool valid = (ow < p.OW) && (oh < p.OH) && (n < p.N);
            const size_t pix = ((size_t)n * p.OHF + (size_t)oh * p.os + p.ooh) * p.OWF + (size_t)ow * p.os + p.oow;
            const float* t_row = acc_tile + (size_t)r * p.acc_ld;
            if (p.epi == 0) {
                const int cols_half = p.BN >> 1;
                float ps = 1.f, pm = 1.f, om_hair = 0.f, om_back = 1.f;
                if (valid) {
                    if (p.pscale) ps = __ldg(p.pscale + pix);
                    if (p.pmul) pm = __ldg(p.pmul + pix);
                    if (p.bf) {
                        const size_t mp = ((size_t)n * p.MH + (size_t)oh * p.mask_stride) * p.MW +
                                          (size_t)ow * p.mask_stride;
                        om_hair = 1.f - __ldg(p.hair + mp);
                        om_back = 1.f - __ldg(p.back + mp);
                    }
                }
                const float* resp = nullptr;
                if (p.res && valid)
                    resp = p.res + (((size_t)n * p.RH + (oh >> p.res_shift)) * p.RW + (ow >> p.res_shift)) * p.Cout;
                for (int j0 = half * cols_half; j0 < (half + 1) * cols_half; j0 += 16) {
                    uint32_t v[16];
                    acc_ld16(t_row, j0, v);
                    const int c0 = nt * p.BN + j0;
                    if (valid && c0 < p.Cout) {
                        float y[16];
#pragma unroll
                        for (int i = 0; i < 16; ++i) y[i] = __uint_as_float(v[i]) * ps;
                        if (p.bias) {
#pragma unroll
                            for (int i = 0; i < 16; i += 4) {
                                const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + c0 + i));
                                y[i] += b.x; y[i + 1] += b.y; y[i + 2] += b.z; y[i + 3] += b.w;
                            }
                        }
                        if (resp) {
#pragma unroll
                            for (int i = 0; i < 16; i += 4) {
                                const float4 b = __ldg(reinterpret_cast<const float4*>(resp + c0 + i));
                                y[i] += b.x; y[i + 1] += b.y; y[i + 2] += b.z; y[i + 3] += b.w;
                            }
                        }
#pragma unroll
                        for (int i = 0; i < 16; ++i) y[i] = apply_act(y[i], p.act);
                        if (p.bf) {
                            const float* bfp = p.bf + pix * p.Cout + c0;
#pragma unroll
                            for (int i = 0; i < 16; i += 4) {
                                const float4 b = __ldg(reinterpret_cast<const float4*>(bfp + i));
                                y[i] = b.x * om_hair + y[i] * om_back;
                                y[i + 1] = b.y * om_hair + y[i + 1] * om_back;
                                y[i + 2] = b.z * om_hair + y[i + 2] * om_back;
                                y[i + 3] = b.w * om_hair + y[i + 3] * om_back;
                            }
                        }
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            y[i] *= pm;
                            if (p.round_out) y[i] = round_tf32(y[i]);
                        }
                        if (p.out) {
                            float4* op = reinterpret_cast<float4*>(p.out + pix * p.Cout + c0);
                            if (p.accumulate) {
#pragma unroll
                                for (int i = 0; i < 4; ++i) {
                                    const float4 o = op[i];
                                    y[4 * i] += o.x; y[4 * i + 1] += o.y; y[4 * i + 2] += o.z; y[4 * i + 3] += o.w;
                                }
                            }
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                op[i] = make_float4(y[4 * i], y[4 * i + 1], y[4 * i + 2], y[4 * i + 3]);
                        }
                        if (p.out_hi) store16(p, y, pix * p.Cout + c0);
                    }
                }
            } else {
                // SPADE: columns [0,BN/2) = gamma, [BN/2,BN) = beta of channels nt*BN/2 + j
                const int ch_tile = p.BN >> 1;
                const int ch_half = ch_tile >> 1;
                const float* xp = nullptr;
                if (valid)
                    xp = p.x + (((size_t)n * p.XH + (oh >> p.x_shift)) * p.XW + (ow >> p.x_shift)) * p.Cout;
                for (int j0 = half * ch_half; j0 < (half + 1) * ch_half; j0 += 16) {
                    uint32_t g[16], b[16];
                    acc_ld16(t_row, j0, g);
                    acc_ld16(t_row, ch_tile + j0, b);
                    const int c0 = nt * ch_tile + j0;
                    if (valid && c0 < p.Cout) {
                        float y[16];
#pragma unroll
                        for (int i = 0; i < 16; i += 4) {
                            const float4 xv = __ldg(reinterpret_cast<const float4*>(xp + c0 + i));
                            const float4 sc = __ldg(reinterpret_cast<const float4*>(p.nscale + c0 + i));
                            const float4 sh = __ldg(reinterpret_cast<const float4*>(p.nshift + c0 + i));
                            const float4 g1 = __ldg(reinterpret_cast<const float4*>(p.gbias1 + c0 + i));
                            const float4 bb = __ldg(reinterpret_cast<const float4*>(p.bbias + c0 + i));
                            const float4 gs = make_float4(g1.x + __uint_as_float(g[i]), g1.y + __uint_as_float(g[i + 1]),
                                                          g1.z + __uint_as_float(g[i + 2]), g1.w + __uint_as_float(g[i + 3]));
                            if (p.aux) *reinterpret_cast<float4*>(p.aux + pix * p.Cout + c0 + i) = gs;  // 1+gamma, kept for backward
                            y[i] = fmaf(fmaf(xv.x, sc.x, sh.x), gs.x, bb.x + __uint_as_float(b[i]));
                            y[i + 1] = fmaf(fmaf(xv.y, sc.y, sh.y), gs.y, bb.y + __uint_as_float(b[i + 1]));
                            y[i + 2] = fmaf(fmaf(xv.z, sc.z, sh.z), gs.z, bb.z + __uint_as_float(b[i + 2]));
                            y[i + 3] = fmaf(fmaf(xv.w, sc.w, sh.w), gs.w, bb.w + __uint_as_float(b[i + 3]));
                        }
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            y[i] = apply_act(y[i], p.act);
                            if (p.round_out) y[i] = round_tf32(y[i]);
                        }
                        if (p.out) {
                            float4* op = reinterpret_cast<float4*>(p.out + pix * p.Cout + c0);
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                op[i] = make_float4(y[4 * i], y[4 * i + 1], y[4 * i + 2], y[4 * i + 3]);
                        }
                        if (p.out_hi) store16(p, y, pix * p.Cout + c0);
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
struct IgemmLaunch {
    const CUtensorMap *tmA, *tmA2, *tmB;
    const IgemmParams* p;
    int grid;
    size_t smem_bytes;
    cudaStream_t stream;
    template <int FMT, int BN, bool MERGED, int SPEC, int CW>
    int run() const {
        if constexpr (conv_variant_exists<FMT, BN, MERGED, SPEC, CW>()) {
            static thread_local int attr_dev = -1;
            return launch_conv_kernel(igemm_tf32_kernel<FMT, BN, MERGED, SPEC, CW>, attr_dev, grid, smem_bytes, stream, *tmA, *tmA2,
                                      *tmB, *p);
        } else {
            return set_error(-14, "mg_conv_igemm: no kernel variant for format %d, BN %d, merged %d, SPEC %d, CW %d", FMT, BN,
                             (int)MERGED, SPEC, CW);
        }
    }
};

static int next_pow2(int v) {
    int r = 1;
    while (r < v) r <<= 1;
    return r;
}

int igemm_launch(const mg_igemm_args* a, cudaStream_t stream) {
    if (!a || !a->in || !a->wpack || (!a->out && !a->out_hi)) return set_error(-1, "mg_conv_igemm: null pointer");
    if (a->a_fmt < 0 || a->a_fmt > 2) return set_error(-9, "mg_conv_igemm: a_fmt must be 0 (tf32), 1 (fp16) or 2 (bf16)");
    const int kelem = a->a_fmt == 0 ? 32 : 64;
    if (a->Cin % kelem != 0)
        return set_error(-2, "mg_conv_igemm: Cin must be a multiple of %d (got %d)", kelem, a->Cin);
    if (a->split && (a->a_fmt == 0 || !a->in_lo)) return set_error(-10, "mg_conv_igemm: split precision needs 16-bit operands and in_lo");
    if (a->out_hi && (a->out16_fmt < 1 || a->out16_fmt > 2)) return set_error(-11, "mg_conv_igemm: out16_fmt must be 1 or 2");
    if (a->out_lo && !a->out_hi) return set_error(-12, "mg_conv_igemm: out_lo without out_hi");
    const int coutg = a->epi == MG_EPI_SPADE ? 2 * a->Cout : a->Cout;
    // BN: 32, 64 or 128 accumulator columns (the wgmma N of the consumer warpgroups; 128 keeps the accumulator at 64 registers
    // per thread and its smem tile at 66 KB).  A wider request is narrowed.
    int BN = a->BN == 0 || a->BN > kMaxAccCols ? kMaxAccCols : a->BN;
    while (BN > 32 && coutg % BN != 0) BN /= 2;
    if (a->BN == 0 && a->epi != MG_EPI_SPADE && tune(TK_BN_FILL)) {
        // Under-filled grids (the 8x8 .. 32x32 layers: 1024 -> 1024 at 8x8 is 4 pixel tiles x 8 column tiles = 32 CTAs on 132
        // SMs): halve BN while twice as many tiles still fit one wave.  Thinner tiles cost MMA efficiency, idle SMs cost more.
        // The weight operand layout does not depend on BN.
        const int tw = next_pow2(a->OW) < 16 ? next_pow2(a->OW) : 16;
        const int th = next_pow2(a->OH) < 128 / tw ? next_pow2(a->OH) : 128 / tw;
        const int tn = 128 / (tw * th);
        const long long m_tiles = (long long)((a->OW + tw - 1) / tw) * ((a->OH + th - 1) / th) * ((a->N + tn - 1) / tn);
        while (BN > 64 && coutg % (BN / 2) == 0 && m_tiles * (coutg / BN) * 2 <= num_sms()) BN /= 2;
    }
    if (BN != 32 && BN != 64 && BN != 128) return set_error(-3, "mg_conv_igemm: bad BN %d", BN);
    if (coutg % BN != 0) return set_error(-4, "mg_conv_igemm: GEMM N %d not a multiple of BN %d", coutg, BN);
    if (a->epi == MG_EPI_SPADE && (BN % 64 != 0 || !a->x || !a->nscale || !a->nshift || !a->gbias1 || !a->bbias))
        return set_error(-5, "mg_conv_igemm: SPADE epilogue needs x/nscale/nshift/gbias1/bbias and BN%%64==0");
    if (a->stride < 1 || a->stride > 2) return set_error(-6, "mg_conv_igemm: stride must be 1 or 2");
    if ((a->bf != nullptr) && (!a->hair || !a->back)) return set_error(-7, "mg_conv_igemm: blend needs hair/back");

    IgemmParams p;
    memset(&p, 0, sizeof(p));
    p.N = a->N; p.OH = a->OH; p.OW = a->OW; p.Cout = a->Cout;
    p.Cin = a->Cin; p.KH = a->KH; p.KW = a->KW; p.stride = a->stride;
    p.pad_h = a->pad + a->pad_h_extra; p.pad_w = a->pad + a->pad_w_extra;
    p.os = a->out_stride > 0 ? a->out_stride : 1; p.ooh = a->out_off_h; p.oow = a->out_off_w;
    p.OHF = a->OHF > 0 ? a->OHF : a->OH; p.OWF = a->OWF > 0 ? a->OWF : a->OW; p.accumulate = a->accumulate;
    if (p.os != 1 && (a->epi != MG_EPI_BIAS || a->res || a->bf || a->pscale || a->pmul))
        return set_error(-8, "mg_conv_igemm: strided output supports the plain bias epilogue only");
    const int epi_impl_env = a->epi == MG_EPI_SPADE ? tune(TK_EPI_IMPL_SPADE) : tune(TK_EPI_IMPL);
    // epilogue chunk width: 16 channels (no register spills) unless MG_EPI_CW16=0 / MG_EPI_CW_SPADE=32 ask for 32
    const int epi_cw16_env = tune(TK_EPI_CW16);
    p.epi_impl = epi_impl_env; p.epi_cw16 = epi_cw16_env;
    // epilogue chunk width (channels per accumulator->scratch->register round): 16 everywhere by default (no register spills,
    // 20 KB of scratch); MG_EPI_CW16=0 / MG_EPI_CW_SPADE=32 select 32 where possible.
    const int span_epi = a->epi == MG_EPI_SPADE ? (BN >> 2) : (BN >> 1);
    const int cw_spade = tune(TK_CW_SPADE);
    int cw = (span_epi % 32 == 0 && !p.epi_cw16) ? 32 : 16;
    if (a->epi == MG_EPI_SPADE) cw = (cw_spade == 32 && span_epi % 32 == 0) ? 32 : 16;
    int scratch_bytes = p.epi_impl == 1 ? kNumEpiWarps * 32 * (cw + 4) * 4 : 0;
    // Halo mode: 3x3 / stride 1 / pad 1 convolutions (the SPADE gamma|beta GEMMs, conv_0/conv_1 and their dgrads) load
    // one [PW x (TH+2)] input patch per K chunk and read the 9 taps out of it through shifted wgmma descriptors.
    // MG_HALO: 0 off (default), 1 on; MG_HALO_PW: patch pitch in pixels (10 = exact, 16 = swizzle-atom aligned rows).
    const int halo_env = tune(TK_HALO);
    const int halo_pw = tune(TK_HALO_PW);
    bool halo = halo_env && p.epi_impl == 1 && a->KH == 3 && a->KW == 3 && a->stride == 1 && p.pad_h == 1 && p.pad_w == 1 &&
                a->OH >= 16 && a->OW >= 8 && a->H == a->OH && a->W == a->OW && (halo_pw == 10 || halo_pw == 16);
    // merged split precision: A_hi x [W_hi ; W_lo] (N = 2*BN) + A_lo x W_hi (N = BN): two MMAs per K step instead of
    // three; the accumulator is 2*BN columns wide and the epilogue adds the halves.  MG_MERGE=0 restores the 3-pass form.
    // Only where 2*BN still fits the accumulator.
    const int merge_env = tune(TK_MERGE);
    bool merged = false;
    if (a->split && merge_env && p.epi_impl == 1 && 2 * BN <= kMaxAccCols) merged = true;
    if (halo && a->split && !merged) halo = false;
    p.halo = halo ? 1 : 0;
    p.merged = merged ? 1 : 0;
    if (halo) { p.TW = 8; p.TH = 16; p.TN = 1; }
    else {
        p.TW = next_pow2(a->OW) < 16 ? next_pow2(a->OW) : 16;
        int th = 128 / p.TW;
        p.TH = next_pow2(a->OH) < th ? next_pow2(a->OH) : th;
        p.TN = 128 / (p.TW * p.TH);
    }
    p.tiles_w = (a->OW + p.TW - 1) / p.TW;
    p.tiles_h = (a->OH + p.TH - 1) / p.TH;
    p.tiles_n = (a->N + p.TN - 1) / p.TN;
    p.BN = BN;
    p.n_tiles = coutg / BN;
    p.num_tiles = p.tiles_w * p.tiles_h * p.tiles_n * p.n_tiles;
    p.kchunks = a->Cin / kelem;
    p.a_fmt = a->a_fmt; p.parts = merged ? 2 : (a->split ? 3 : 1); p.kelem = kelem;
    p.out_hi = a->out_hi; p.out_lo = a->out_lo; p.out16_fmt = a->out16_fmt;
    p.acc_cols = p.merged ? 2 * BN : BN;
#ifdef MG_PROBES
    p.dbg = probe_bits();
#endif
    const int stage_bytes = kABytes + p.acc_cols * 128;
    p.acc_ld = p.acc_cols + 4;
    const int acc_bytes = 128 * p.acc_ld * 4;
    const int smem_avail = 227 * 1024 - 1024 - 512 - scratch_bytes - acc_bytes;
    size_t ring_bytes = 0;
    if (halo) {
        p.PW = halo_pw;
        p.patch_tx = p.PW * (p.TH + 2) * 128;
        p.patch_bytes = (p.patch_tx + 1023) & ~1023;
        p.b_slot_bytes = p.acc_cols * 128;
        p.n_items = p.kchunks * (p.merged ? 2 : 1);
        p.a_slots = 2;
        p.b_slots = (smem_avail - p.a_slots * p.patch_bytes) / p.b_slot_bytes;
        if (p.b_slots > kMaxStages) {   // room to spare: deepen the patch ring first
            p.a_slots = 3;
            p.b_slots = (smem_avail - p.a_slots * p.patch_bytes) / p.b_slot_bytes;
            if (p.b_slots > kMaxStages) p.b_slots = kMaxStages;
        }
        // the consumers hold two weight slots (the step in flight and the one being issued): a third keeps the producer busy
        if (p.b_slots < 3) return set_error(-13, "mg_conv_igemm: halo rings do not fit shared memory");
        ring_bytes = (size_t)p.a_slots * p.patch_bytes + (size_t)p.b_slots * p.b_slot_bytes;
        p.stages = p.b_slots;
    } else {
        int stages = smem_avail / stage_bytes;
        if (stages > kMaxStages) stages = kMaxStages;
        const int stages_cap = tune(TK_STAGES);
        if (stages_cap > 0 && stages > stages_cap) stages = stages_cap > 3 ? stages_cap : 3;
        // the consumers hold two stages (the step in flight and the one being issued): a third keeps the producer busy
        if (stages < 3) return set_error(-13, "mg_conv_igemm: stage ring does not fit shared memory");
        p.stages = stages;
        ring_bytes = (size_t)stages * stage_bytes;
    }
    p.bar_off = (int)ring_bytes;
    p.epi_off = (int)ring_bytes + 512;
    p.acc_off = p.epi_off + scratch_bytes;
    p.epi = a->epi; p.act = a->act; p.round_out = a->round_out;
    p.out = a->out; p.bias = a->bias;
    p.res = a->res; p.res_shift = a->res_shift;
    p.RH = a->OH >> a->res_shift; p.RW = a->OW >> a->res_shift;
    p.pscale = a->pscale; p.pmul = a->pmul;
    p.bf = a->bf; p.hair = a->hair; p.back = a->back;
    p.mask_stride = a->mask_stride; p.MH = a->MH; p.MW = a->MW;
    p.x = a->x; p.x_shift = a->x_shift; p.XH = a->OH >> a->x_shift; p.XW = a->OW >> a->x_shift;
    p.nscale = a->nscale; p.nshift = a->nshift; p.gbias1 = a->gbias1; p.bbias = a->bbias; p.aux = a->aux_out;

    int spec = 0;
    if (p.epi_impl >= 1 && a->epi == MG_EPI_SPADE && !a->out && a->out_hi && a->out_lo && a->out16_fmt == 2 && !a->aux_out &&
        !a->round_out && (a->act == MG_ACT_LRELU || a->act == MG_ACT_NONE))
        spec = a->act == MG_ACT_LRELU ? 1 : 2;
    // 3x3 / stride 1 / pad 1 layers: the halo-patch + M-tile-group kernel (mg_conv3x3.cu) moves 3-5x fewer bytes through L2.
    // MG_GROUP3: 0 off, 1 or 2 (default 1) every eligible layer.
    {
        const int g3 = tune(TK_GROUP3);
        if (!halo && g3) {
            IgemmParams p3 = p;
            const int rc3 = conv3x3_group_launch(a, p3, BN, cw, scratch_bytes, spec, stream);
            if (rc3 == 1) return 0;
            if (rc3 != 0) return rc3;
        }
    }

    CUtensorMap tmA, tmA2, tmB;
    const int esz = a->a_fmt == 0 ? 4 : 2;
    const CUtensorMapDataType dt = a->a_fmt == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : a->a_fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    {
        cuuint64_t dims[4] = {(cuuint64_t)a->Cin, (cuuint64_t)a->W, (cuuint64_t)a->H, (cuuint64_t)a->N};
        cuuint64_t strides[3] = {(cuuint64_t)a->Cin * esz, (cuuint64_t)a->W * a->Cin * esz,
                                 (cuuint64_t)a->H * a->W * a->Cin * esz};
        cuuint32_t box[4] = {(cuuint32_t)kelem, (cuuint32_t)(p.TW * a->stride), (cuuint32_t)(p.TH * a->stride), (cuuint32_t)p.TN};
        if (halo) { box[1] = (cuuint32_t)p.PW; box[2] = (cuuint32_t)(p.TH + 2); box[3] = 1; }
        cuuint32_t estr[4] = {1, (cuuint32_t)a->stride, (cuuint32_t)a->stride, 1};
        int rc = encode_tensor_map(&tmA, (void*)a->in, dt, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
        rc = encode_tensor_map(&tmA2, (void*)(a->split ? a->in_lo : a->in), dt, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    {
        const cuuint64_t ktot = (cuuint64_t)a->KH * a->KW * a->Cin * (a->split ? 2 : 1);
        cuuint64_t dims[2] = {ktot, (cuuint64_t)coutg};
        cuuint64_t strides[1] = {ktot * esz};
        cuuint32_t box[2] = {(cuuint32_t)kelem, (cuuint32_t)BN};
        cuuint32_t estr[2] = {1, 1};
        int rc = encode_tensor_map(&tmB, (void*)a->wpack, dt, 2, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const size_t smem_bytes = ring_bytes + 1024 /*align slack*/ + 512 /*barriers*/ + scratch_bytes + acc_bytes;
    int grid = num_sms();
    if (a->max_ctas > 0 && a->max_ctas < grid) grid = a->max_ctas;
    if (grid > p.num_tiles) grid = p.num_tiles;
    const IgemmLaunch l{&tmA, &tmA2, &tmB, &p, grid, smem_bytes, stream};
    return dispatch_conv_variant(l, p.a_fmt, BN, merged, spec, cw);
}

}  // namespace mg

extern "C" int mg_conv_igemm(const mg_igemm_args* a, void* stream) {
    return mg::igemm_launch(a, reinterpret_cast<cudaStream_t>(stream));
}
