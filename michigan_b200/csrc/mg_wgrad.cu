// michigan_b200 — weight-gradient implicit GEMM on tensor cores (sm_90a).
//
//   dW[co, tap, ci] = sum_{pixels} dY[pix, co] * X[pix (+) tap, ci]
//
// GEMM view per filter row kh: D[M = 128 output channels, N = KW x BN input channels] accumulated over
// K = pixels.  Both operands are NHWC activations, i.e. contiguous along their M/N index and strided
// along K: MN-major operands.  Every TMA box [pix_tile pixels x 128 B of channels] lands 128B-swizzled.
// bf16: two consumer warpgroups (output channels 0-63 / 64-127 of the M tile) run wgmma with both operands
// transposed straight from those boxes, one accumulator per filter tap (KW x BN columns, KW and BN compile-time).
// TF32: wgmma reads MN-major operands only in 16-bit formats, so the product runs on warp-level mma.sync
// (m16n8k8) with fragments gathered from the stage.  The tap shift and the conv zero
// padding come from the box start coordinate + TMA OOB zero fill, exactly as in the forward kernel.
// Pixels are split across CTAs (split-K); the partial tiles are summed in an fp64 buffer (mg_internal.h:
// acc64_*), so the gradient does not depend on the order in which the splits finish.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include "mg_ptx.cuh"
#include "mg_internal.h"

namespace mg {

// warps 0-7: consumers (output channels 16*warp.. of the M tile, all KW x BN columns), warp 8: TMA producer
constexpr int kWgThreads = 288;
constexpr int kWgStagesMax = 6;
constexpr int kWgMaxCols = 256;   // KW x BN accumulator columns: 128 fp32 registers per consumer thread

struct WgradParams {
    int N, OH, OW, Cout, Cin, KH, KW, stride, pad;
    int TW, TH, TN, tiles_w, tiles_h, tiles_n, pix_tiles;
    int BN, m_tiles, n_tiles, splits, stages;
    int pix_tile, box_bytes;   // K (pixels) per pipeline stage: 32 or 64; bytes of one [pix_tile x 128 B] box
    int f16;                   // 0: fp32 storage read as TF32 (32 channels per 128 B row, K = 8 pixels per MMA);
                               // 2: bf16 operands (64 channels per row, K = 16 pixels per MMA)
    int kelem, mboxes, kmma;   // channels per box, boxes per 128-row M tile, pixels per MMA
    float* dw;      // [Cout][KH*KW*Cin]
    double* dw64;   // same layout, fp64 sum of the splits (splits > 1)
};

// byte offset of (pixel row k, byte b of the 128 B channel row) inside a 1024 B-aligned SWIZZLE_128B box
__device__ __forceinline__ uint32_t sw128(uint32_t k, uint32_t b) {
    const uint32_t o = k * 128 + b;
    return o ^ ((k & 7) << 4);
}

__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_bf16_16x8x16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// KWT > 0: the bf16 wgmma consumer for KW = KWT taps of BN = BNT channels; KWT == 0: the mma.sync consumer (any format).
template <int KWT, int BNT>
__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_tf32_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WgradParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    // One unit = one filter ROW (kh): the dY tile is loaded once per stage and multiplied with the KW shifted
    // input tiles (accumulator columns kw*BN..), so dY is streamed KH (not KH*KW) times from HBM/L2.
    const int kBoxBytes = p.box_bytes;
    const int a_bytes = p.mboxes * kBoxBytes;           // M = 128 -> 4 boxes of 32 fp32 channels / 2 boxes of 64 bf16 channels
    const int b1_bytes = (p.BN / p.kelem) * kBoxBytes;  // one tap's input tile
    const int stage_bytes = a_bytes + p.KW * b1_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + kWgStagesMax;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // unit decode: blockIdx.x = split * units + (kh * m_tiles + mt) * n_tiles + nt
    // units are the FAST index: the CTAs of one wave work on the same pixel range, so dY / X come from DRAM once per wave
    const int n_units = p.KH * p.m_tiles * p.n_tiles;
    int u = blockIdx.x % n_units;
    const int split = blockIdx.x / n_units;
    const int nt = u % p.n_tiles; u /= p.n_tiles;
    const int mt = u % p.m_tiles;
    const int kh = u / p.m_tiles;
    const int t_begin = (int)((long long)p.pix_tiles * split / p.splits);
    const int t_end = (int)((long long)p.pix_tiles * (split + 1) / p.splits);

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmDY);
        tma_prefetch_desc(&tmX);
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        // TMA producer WARP: a stage is mboxes + KW*(BN/kelem) boxes of [pix_tile x 128 B]; lane j issues box j, so a stage
        // goes out in one pass.
        int st = 0; uint32_t ph = 0;
        const int nb_x = p.BN / p.kelem;
        const uint32_t tx = (uint32_t)stage_bytes;
        const int n_boxes = p.mboxes + p.KW * nb_x;
        for (int t = t_begin; t < t_end; ++t) {
            const int tw = t % p.tiles_w;
            const int th = (t / p.tiles_w) % p.tiles_h;
            const int tn = t / (p.tiles_w * p.tiles_h);
            const int ow0 = tw * p.TW, oh0 = th * p.TH, n0 = tn * p.TN;
            if (lane == 0) {
                mbar_wait_report(&empty_bar[st], ph ^ 1);
                mbar_arrive_expect_tx(&full_bar[st], tx);
            }
            __syncwarp();
            uint8_t* sa = smem + (size_t)st * stage_bytes;
            for (int b = lane; b < n_boxes; b += 32) {
                if (b < p.mboxes) {
                    tma_load_4d(sa + b * kBoxBytes, &tmDY, &full_bar[st], mt * 128 + b * p.kelem, ow0, oh0, n0);
                } else {
                    const int kw = (b - p.mboxes) / nb_x, j = (b - p.mboxes) - kw * nb_x;
                    tma_load_4d(sa + a_bytes + kw * b1_bytes + j * kBoxBytes, &tmX, &full_bar[st], nt * p.BN + j * p.kelem,
                                ow0 * p.stride - p.pad + kw, oh0 * p.stride - p.pad + kh, n0);
                }
            }
            __syncwarp();
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
    } else if constexpr (KWT > 0) {
        // Consumer warpgroup wg: output channels 64*wg.. (= dY box wg) x KW taps of BN input channels, one register
        // accumulator per tap; K step = 16 pixel rows = 2048 B of every box.
        const int wg = warp >> 2;
        float acc[KWT][BNT / 2];
#pragma unroll
        for (int kw = 0; kw < KWT; ++kw)
#pragma unroll
            for (int i = 0; i < BNT / 2; ++i) acc[kw][i] = 0.f;
        int st = 0; uint32_t ph = 0;
        for (int t = t_begin; t < t_end; ++t) {
            mbar_wait(&full_bar[st], ph);
            const uint32_t sa = smem_u32(smem + (size_t)st * stage_bytes);
            const uint32_t a_base = sa + (uint32_t)(wg * kBoxBytes), b_base = sa + (uint32_t)a_bytes;
            wgmma_fence();
#pragma unroll 1
            for (int kk = 0; kk < p.pix_tile; kk += 16) {
                const uint64_t da = wg_desc_mn_sw128(a_base + (uint32_t)(kk * 128), (uint32_t)kBoxBytes);
#pragma unroll
                for (int kw = 0; kw < KWT; ++kw) {
                    const uint64_t db = wg_desc_mn_sw128(b_base + (uint32_t)(kw * b1_bytes + kk * 128), (uint32_t)kBoxBytes);
                    if constexpr (BNT == 128) wgmma_bf16_tt_n128(acc[kw], da, db, 1u);
                    else wgmma_bf16_tt_n64(acc[kw], da, db, 1u);
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[st]);
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
        if (t_end > t_begin) {
            // wgmma layout: warp w of the warpgroup owns rows 16w..16w+15; register 4j+{0,1} = row lane/4, columns
            // 8j + 2(lane%4) + {0,1}; register 4j+{2,3} = the same columns 8 rows further down
            const int r0 = mt * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = (lane & 3) * 2;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int co = r0 + 8 * h;
                if (co >= p.Cout) continue;
#pragma unroll
                for (int kw = 0; kw < KWT; ++kw)
#pragma unroll
                    for (int j = 0; j < BNT / 8; ++j) {
                        const size_t off = (size_t)co * (p.KH * KWT * p.Cin) + (size_t)(kh * KWT + kw) * p.Cin + nt * BNT + j * 8 + c0;
                        const float v0 = acc[kw][4 * j + 2 * h], v1 = acc[kw][4 * j + 2 * h + 1];
                        if (p.splits > 1) {
                            atomicAdd(p.dw64 + off, (double)v0);
                            atomicAdd(p.dw64 + off + 1, (double)v1);
                        } else {
                            *reinterpret_cast<float2*>(p.dw + off) = make_float2(v0, v1);
                        }
                    }
            }
        }
    } else {
        // Consumer warp: rows m0.. m0+15 (output channels) x all KW*BN columns, one m16n8 accumulator per 8 columns.
        // Fragments (g = lane / 4, t = lane % 4): A[m][k] = dY tile (pixel row k, channel m), B[k][n] = X tile (pixel row k, channel n).
        const int g = lane >> 2, t4 = lane & 3;
        const int m0 = warp * 16;
        const int ncols = p.KW * p.BN, n8 = ncols >> 3;
        const int esz = p.f16 ? 2 : 4;
        // per-thread smem byte offsets of the two A rows (channels m0+g, m0+g+8) and of this thread's B column in each n8 tile
        uint32_t a_off[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + g + 8 * h;
            a_off[h] = (uint32_t)((m / p.kelem) * kBoxBytes) | ((uint32_t)((m % p.kelem) * esz) << 20);
        }
        float acc[kWgMaxCols / 8][4];
#pragma unroll
        for (int j = 0; j < kWgMaxCols / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        int st = 0; uint32_t ph = 0;
        for (int t = t_begin; t < t_end; ++t) {
            mbar_wait(&full_bar[st], ph);
            const uint8_t* sa = smem + (size_t)st * stage_bytes;
            auto ldA = [&](int h, int k) -> const uint8_t* { return sa + (a_off[h] & 0xFFFFF) + sw128(k, a_off[h] >> 20); };
            for (int kk = 0; kk < p.pix_tile; kk += p.kmma) {
                uint32_t a[4];
                if (p.f16) {
                    // a0 = A[g][kk+2t..+1], a1 = A[g+8][..], a2 = A[g][kk+2t+8..+9], a3 = A[g+8][..]
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int h = i & 1, k = kk + 2 * t4 + 8 * (i >> 1);
                        a[i] = (uint32_t)*reinterpret_cast<const uint16_t*>(ldA(h, k)) |
                               ((uint32_t)*reinterpret_cast<const uint16_t*>(ldA(h, k + 1)) << 16);
                    }
                } else {
                    // a0 = A[g][kk+t], a1 = A[g+8][kk+t], a2 = A[g][kk+t+4], a3 = A[g+8][kk+t+4]
#pragma unroll
                    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const uint32_t*>(ldA(i & 1, kk + t4 + 4 * (i >> 1)));
                }
#pragma unroll
                for (int j = 0; j < kWgMaxCols / 8; ++j) {
                    if (j < n8) {
                        const int n = j * 8 + g, kw = n / p.BN, ci = n - kw * p.BN;
                        const uint8_t* bb = sa + a_bytes + kw * b1_bytes + (ci / p.kelem) * kBoxBytes;
                        const uint32_t cb = (uint32_t)((ci % p.kelem) * esz);
                        if (p.f16) {
                            // b0 = B[kk+2t..+1][n], b1 = B[kk+2t+8..+9][n]
                            const int k = kk + 2 * t4;
                            const uint32_t b0 = (uint32_t)*reinterpret_cast<const uint16_t*>(bb + sw128(k, cb)) |
                                                ((uint32_t)*reinterpret_cast<const uint16_t*>(bb + sw128(k + 1, cb)) << 16);
                            const uint32_t b1 = (uint32_t)*reinterpret_cast<const uint16_t*>(bb + sw128(k + 8, cb)) |
                                                ((uint32_t)*reinterpret_cast<const uint16_t*>(bb + sw128(k + 9, cb)) << 16);
                            mma_bf16_16x8x16(acc[j], a, b0, b1);
                        } else {
                            // b0 = B[kk+t][n], b1 = B[kk+t+4][n]
                            const uint32_t b0 = *reinterpret_cast<const uint32_t*>(bb + sw128(kk + t4, cb));
                            const uint32_t b1 = *reinterpret_cast<const uint32_t*>(bb + sw128(kk + t4 + 4, cb));
                            mma_tf32_16x8x8(acc[j], a, b0, b1);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[st]);
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
        if (t_end > t_begin) {
            // c0,c1 = (row g, columns 2t, 2t+1), c2,c3 = (row g+8, same columns)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int co = mt * 128 + m0 + g + 8 * h;
                if (co >= p.Cout) continue;
#pragma unroll
                for (int j = 0; j < kWgMaxCols / 8; ++j) {
                    if (j < n8) {
                        const int n = j * 8 + 2 * t4, kw = n / p.BN, ci = n - kw * p.BN;
                        const size_t off = (size_t)co * (p.KH * p.KW * p.Cin) + (size_t)(kh * p.KW + kw) * p.Cin + nt * p.BN + ci;
                        if (p.splits > 1) {
                            atomicAdd(p.dw64 + off, (double)acc[j][2 * h]);
                            atomicAdd(p.dw64 + off + 1, (double)acc[j][2 * h + 1]);
                        } else {
                            *reinterpret_cast<float2*>(p.dw + off) = make_float2(acc[j][2 * h], acc[j][2 * h + 1]);
                        }
                    }
                }
            }
        }
    }
}

static int np2(int v) { int r = 1; while (r < v) r <<= 1; return r; }

}  // namespace mg

using namespace mg;

// dw: [Cout][KH*KW*Cin] fp32 (tap-major K, the layout of mg_pack_weight); overwritten.
// fmt 0: dy / x fp32 (read as TF32); fmt 2: dy / x bf16.
static int wgrad_launch(const void* dy, const void* x, float* dw, int N, int H, int W, int Cin, int OH, int OW, int Cout,
                        int KH, int KW, int stride, int pad, int fmt, cudaStream_t stream) {
    if (!dy || !x || !dw) return set_error(-1, "mg_conv_wgrad: null pointer");
    if (fmt != 0 && fmt != 2) return set_error(-5, "mg_conv_wgrad: operand format must be 0 (tf32) or 2 (bf16)");
    const int kelem = fmt ? 64 : 32;
    if (Cin % kelem != 0 || Cout % kelem != 0) return set_error(-2, "mg_conv_wgrad: channels must be multiples of %d", kelem);
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.N = N; p.OH = OH; p.OW = OW; p.Cout = Cout; p.Cin = Cin; p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad;
    p.f16 = fmt; p.kelem = kelem; p.mboxes = 128 / kelem; p.kmma = fmt ? 16 : 8;
    int BN = Cin >= 128 ? 128 : Cin;
    if (Cin % BN != 0) BN = kelem;
    while (KW * BN > kWgMaxCols) BN /= 2;                // KW accumulators of BN columns must fit the consumer registers
    if (BN < kelem || Cin % BN != 0) return set_error(-3, "mg_conv_wgrad: KW %d x Cin %d does not fit the accumulator", KW, Cin);
    p.BN = BN;
    // K (pixels) per stage: 64 when at least 3 stages fit in shared memory, else 32
    int pix_tile = 64;
    if ((200 * 1024) / ((p.mboxes + KW * (BN / kelem)) * 64 * 128) < 3) pix_tile = 32;
    p.pix_tile = pix_tile; p.box_bytes = pix_tile * 128;
    p.TW = np2(OW) < 8 ? np2(OW) : 8;
    int th = pix_tile / p.TW;
    p.TH = np2(OH) < th ? np2(OH) : th;
    p.TN = pix_tile / (p.TW * p.TH);
    p.tiles_w = (OW + p.TW - 1) / p.TW; p.tiles_h = (OH + p.TH - 1) / p.TH; p.tiles_n = (N + p.TN - 1) / p.TN;
    p.pix_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
    p.m_tiles = (Cout + 127) / 128;
    p.n_tiles = Cin / BN;
    const int units = KH * p.m_tiles * p.n_tiles;
    // split-K so that units * splits fills whole waves of one CTA per SM: round DOWN (296 / 6 units = 49 -> 294 CTAs = 2 waves;
    // rounding up gave 300 CTAs = a third wave with 4 CTAs)
    int splits = (2 * num_sms()) / units;
    if (splits < 1) splits = 1;
    if (splits > p.pix_tiles) splits = p.pix_tiles;
    p.splits = splits;
    const int stage_bytes = p.mboxes * p.box_bytes + KW * (BN / kelem) * p.box_bytes;
    int stages = (200 * 1024) / stage_bytes;
    if (stages < 1) return set_error(-4, "mg_conv_wgrad: stage of %d bytes does not fit shared memory", stage_bytes);
    if (stages > kWgStagesMax) stages = kWgStagesMax;
    p.stages = stages;
    p.dw = dw;

    CUtensorMap tmDY, tmX;
    const int esz = fmt ? 2 : 4;
    const CUtensorMapDataType dt = fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
    {
        cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)OW, (cuuint64_t)OH, (cuuint64_t)N};
        cuuint64_t strides[3] = {(cuuint64_t)Cout * esz, (cuuint64_t)OW * Cout * esz, (cuuint64_t)OH * OW * Cout * esz};
        cuuint32_t box[4] = {(cuuint32_t)kelem, (cuuint32_t)p.TW, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
        cuuint32_t es[4] = {1, 1, 1, 1};
        int rc = encode_tensor_map(&tmDY, (void*)dy, dt, 4, dims, strides, box, es, sw);
        if (rc) return rc;
    }
    {
        cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
        cuuint64_t strides[3] = {(cuuint64_t)Cin * esz, (cuuint64_t)W * Cin * esz, (cuuint64_t)H * W * Cin * esz};
        cuuint32_t box[4] = {(cuuint32_t)kelem, (cuuint32_t)(p.TW * stride), (cuuint32_t)(p.TH * stride), (cuuint32_t)p.TN};
        cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
        int rc = encode_tensor_map(&tmX, (void*)x, dt, 4, dims, strides, box, es, sw);
        if (rc) return rc;
    }
    // bf16 with a compiled (KW, BN) pair: the wgmma consumer; otherwise the mma.sync consumer
    void (*kern)(CUtensorMap, CUtensorMap, WgradParams) = wgrad_tf32_kernel<0, 0>;
    if (fmt == 2) {
        if (KW == 1 && BN == 64) kern = wgrad_tf32_kernel<1, 64>;
        else if (KW == 1 && BN == 128) kern = wgrad_tf32_kernel<1, 128>;
        else if (KW == 2 && BN == 64) kern = wgrad_tf32_kernel<2, 64>;
        else if (KW == 2 && BN == 128) kern = wgrad_tf32_kernel<2, 128>;
        else if (KW == 3 && BN == 64) kern = wgrad_tf32_kernel<3, 64>;
        else if (KW == 4 && BN == 64) kern = wgrad_tf32_kernel<4, 64>;
    }
    cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return set_error((int)e, "wgrad attr: %s", cudaGetErrorString(e));
    const size_t smem_bytes = (size_t)stages * stage_bytes + 1024 + 256;
    const size_t n_dw = (size_t)Cout * KH * KW * Cin;
    if (splits > 1) {
        const int rc = acc64_alloc(&p.dw64, n_dw, stream);
        if (rc) return rc;
    }
    kern<<<units * splits, kWgThreads, smem_bytes, stream>>>(tmDY, tmX, p);
    int rc = check_launch("mg_conv_wgrad");
    if (splits > 1) {
        if (!rc) rc = acc64_fold(p.dw64, dw, n_dw, 0, stream);
        const int rc2 = acc64_free(p.dw64, stream);
        if (!rc) rc = rc2;
    }
    return rc;
}

extern "C" int mg_conv_wgrad(const float* dy, const float* x, float* dw, int N, int H, int W, int Cin, int OH, int OW, int Cout,
                             int KH, int KW, int stride, int pad, void* stream_) {
    return wgrad_launch(dy, x, dw, N, H, W, Cin, OH, OW, Cout, KH, KW, stride, pad, 0, reinterpret_cast<cudaStream_t>(stream_));
}

// Same with 16-bit (bf16) operands: dy [N,OH,OW,Cout] and x [N,H,W,Cin] bf16, fp32 accumulation and output.
extern "C" int mg_conv_wgrad16(const void* dy16, const void* x16, float* dw, int N, int H, int W, int Cin, int OH, int OW, int Cout,
                               int KH, int KW, int stride, int pad, void* stream_) {
    return wgrad_launch(dy16, x16, dw, N, H, W, Cin, OH, OW, Cout, KH, KW, stride, pad, 2, reinterpret_cast<cudaStream_t>(stream_));
}
