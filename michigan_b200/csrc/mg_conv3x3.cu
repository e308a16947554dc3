// michigan_b200 — 3x3 / stride 1 / pad 1 implicit-GEMM convolution on wgmma with HALO patches and M-TILE GROUPS.
//
// Why a second kernel.  mg_igemm.cu loads one [128 px x 64 ch] activation box per (tap, K chunk) and streams the whole
// weight operand once per 128-pixel tile: a 3x3 conv therefore pulls 9x its activations plus K*N weights per tile through
// L2: the thin-N layers of the generator (up_3.conv_0, 128 -> 64 at 512^2, bf16 hi+lo) move 17 GB per launch for
// 0.46 PFLOP of MMA work.  Here
//   * ONE [18 x 18 px x 128 B] activation patch per (K chunk, hi|lo part) serves all nine taps of TWO horizontally adjacent
//     M tiles (8 x 16 pixels each) through wgmma descriptors whose start address is shifted by (kh*18 + kw + 8*mt) rows
//     - activation traffic / 7.1;
//   * every weight slot (one tap of one K chunk) is consumed by both M tiles before it is released - weight traffic / 2;
//   * each consumer warpgroup keeps one register accumulator per M tile (2 x 64 registers at 128 columns).
// Same operand formats (TF32 / fp16 / bf16, split precision merged or 3-pass), same epilogues (mg_epilogue.cuh), same
// results as mg_igemm.cu up to accumulation order.
//
// Warp roles (288 threads): warps 0..7 wgmma consumers (rows 0-63 / 64-127 of both M tiles) + epilogue, warp 8 TMA producer.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstring>
#include "mg_ptx.cuh"
#include "mg_internal.h"
#include "mg_epilogue.cuh"

namespace mg {

constexpr int kGM = 2;                 // M tiles per group
constexpr int kPatchW = 8 * kGM + 2;   // 18 pixels
constexpr int kPatchH = 16 + 2;        // 18 rows
constexpr int kPatchTx = kPatchW * kPatchH * 128;
constexpr int kPatchBytes = (kPatchTx + 1023) & ~1023;
constexpr int kMaxBSlots = 8;
constexpr int kASlots = 2;

struct Conv3Params {
    IgemmParams g;          // geometry, operand formats, epilogue (TW = 8, TH = 16, TN = 1)
    int groups_w, num_groups, b_slots, b_slot_bytes, steps_hi, steps_lo, n_items, bar3_off;
};

// item = (K chunk, activation part): part 0 = A (or A_hi), part 1 = A_lo.  Steps of an item = B slots it consumes:
//   plain          : 9 (tap)                                   MMA N = BN
//   merged split   : hi 9 x [W_hi;W_lo] (N = 2BN), lo 9 x W_hi (N = BN)
//   3-pass split   : hi 18 = tap x {W_hi, W_lo} (N = BN),   lo 9 x W_hi (N = BN)
template <int SPEC, int CW>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_group_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                     const __grid_constant__ CUtensorMap tmB, const Conv3Params q) {
    const IgemmParams& p = q.g;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* a_ring = smem;
    uint8_t* b_ring = smem + kASlots * kPatchBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + q.bar3_off);
    uint64_t* bfull = bars;                         // [kMaxBSlots]
    uint64_t* bempty = bars + kMaxBSlots;           // [kMaxBSlots], one arrival per consumer warp
    uint64_t* afull = bars + 2 * kMaxBSlots;        // [kASlots]
    uint64_t* aempty = afull + kASlots;             // [kASlots], one arrival per consumer warp
    float* acc_tile = reinterpret_cast<float*>(smem + p.acc_off);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == kNumEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmA2);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < q.b_slots; ++s) { mbar_init(&bfull[s], 1); mbar_init(&bempty[s], kNumEpiWarps); }
        for (int s = 0; s < kASlots; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], kNumEpiWarps); }
        fence_barrier_init();
    }
    __syncthreads();
    const int groups_per_img = q.groups_w * p.tiles_h;
    const bool split = p.parts > 1;

    if (warp == kNumEpiWarps) {
        // ===================== TMA producer (one thread): A patches are issued one item ahead of the weight stream ===========
        if (lane == 0) {
            int bs = 0, as_ = 0;
            uint32_t bph = 0, aphs = 0;
            // A-patch cursor: runs up to kASlots - 1 items ahead of the weight stream (the next patch is requested as soon as
            // its slot is free, so its L2 latency hides behind the current item's nine-plus weight steps)
            int gia = blockIdx.x, ita = 0;
            long long a_issued = 0, item = 0;
            auto issue_a = [&](bool must) -> bool {
                if (gia >= q.num_groups) return false;
                if (!must && !mbar_test_wait(&aempty[as_], aphs ^ 1)) return false;
                if (must) mbar_wait(&aempty[as_], aphs ^ 1);
                const int mga = gia / p.n_tiles;
                const int gwa = mga % q.groups_w, tha = (mga / q.groups_w) % p.tiles_h, tna = mga / groups_per_img;
                const int kca = split ? (ita >> 1) : ita, parta = split ? (ita & 1) : 0;
                mbar_arrive_expect_tx(&afull[as_], (uint32_t)kPatchTx);
                tma_load_4d(a_ring + (size_t)as_ * kPatchBytes, parta ? &tmA2 : &tmA, &afull[as_], kca * p.kelem, gwa * (8 * kGM) - 1,
                            tha * 16 - 1, tna);
                if (++as_ == kASlots) { as_ = 0; aphs ^= 1; }
                if (++ita == q.n_items) { ita = 0; gia += gridDim.x; }
                ++a_issued;
                return true;
            };
            for (int gi = blockIdx.x; gi < q.num_groups; gi += gridDim.x) {
                const int nt = gi % p.n_tiles;
                for (int it = 0; it < q.n_items; ++it, ++item) {
                    const int kc = split ? (it >> 1) : it, part = split ? (it & 1) : 0;
                    if (a_issued <= item) issue_a(true);
                    const int steps = part ? q.steps_lo : q.steps_hi;
                    for (int st = 0; st < steps; ++st) {
                        if (a_issued < item + kASlots) issue_a(false);
                        // weight K offset: [tap][hi|lo][Cin] when split, [tap][Cin] otherwise
                        int tap, wsel;
                        if (steps == 18) { tap = st >> 1; wsel = st & 1; } else { tap = st; wsel = 0; }
                        const int kofs = (split ? (tap * 2 + wsel) : tap) * p.Cin + kc * p.kelem;
                        mbar_wait(&bempty[bs], bph ^ 1);
                        uint8_t* sb = b_ring + (size_t)bs * q.b_slot_bytes;
                        if (p.merged && part == 0) {
                            mbar_arrive_expect_tx(&bfull[bs], (uint32_t)(2 * p.BN * 128));
                            tma_load_2d(sb, &tmB, &bfull[bs], kofs, nt * p.BN);
                            tma_load_2d(sb + p.BN * 128, &tmB, &bfull[bs], kofs + p.Cin, nt * p.BN);
                        } else {
                            mbar_arrive_expect_tx(&bfull[bs], (uint32_t)(p.BN * 128));
                            tma_load_2d(sb, &tmB, &bfull[bs], kofs, nt * p.BN);
                        }
                        if (++bs == q.b_slots) { bs = 0; bph ^= 1; }
                    }
                }
            }
        }
    } else {
        // ===================== consumers: warpgroup wg multiplies rows 64*wg.. of BOTH M tiles of a group, then all 8 warps
        // run the epilogue of M tile 0 and of M tile 1
        const int wg = warp >> 2;
        const int quarter = warp & 3;
        const int half = warp >> 2;
        float* scr = reinterpret_cast<float*>(smem + p.epi_off) + warp * (32 * (CW + 4));
        const uint32_t a_base0 = smem_u32(a_ring), b_base0 = smem_u32(b_ring);
        float acc0[64], acc1[64];
        int bs = 0, as_ = 0;
        uint32_t bph = 0, aphs = 0;
        for (int gi = blockIdx.x; gi < q.num_groups; gi += gridDim.x) {
            const int nt = gi % p.n_tiles;
            const int mg = gi / p.n_tiles;
            const int gw = mg % q.groups_w, th = (mg / q.groups_w) % p.tiles_h, tn = mg / groups_per_img;
            for (int it = 0; it < q.n_items; ++it) {
                const int part = split ? (it & 1) : 0;
                const int n = (p.merged && part == 1) ? p.BN : p.acc_cols;
                mbar_wait(&afull[as_], aphs);
                // rows 64.. of an M tile are its pixel rows 8.., eight patch rows further on
                const uint32_t a_base = a_base0 + (uint32_t)(as_ * kPatchBytes) + (uint32_t)(wg * 8 * kPatchW * 128);
                const int steps = part ? q.steps_lo : q.steps_hi;
                for (int st = 0; st < steps; ++st) {
                    const int tap = steps == 18 ? (st >> 1) : st;
                    const int kh = tap / 3, kw = tap - kh * 3;
                    mbar_wait(&bfull[bs], bph);
                    // tap (kh, kw) of M tile mt = the patch read from row kh*18 + kw + 8*mt on; 8-pixel row groups are 18 rows apart
                    const uint32_t a_tap = a_base + (uint32_t)((kh * kPatchW + kw) * 128);
                    const uint64_t db = wg_desc_sw128(b_base0 + (uint32_t)(bs * q.b_slot_bytes), 1024);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint32_t accum = (it | st | k) != 0 ? 1u : 0u;
                        const uint64_t da0 = wg_desc_sw128(a_tap + (uint32_t)(k * 32), (uint32_t)(kPatchW * 128));
                        const uint64_t da1 = wg_desc_sw128(a_tap + (uint32_t)(8 * 128 + k * 32), (uint32_t)(kPatchW * 128));
                        wgmma_k32b(acc0, n, p.a_fmt, da0, db + (uint64_t)(2 * k), accum);
                        wgmma_k32b(acc1, n, p.a_fmt, da1, db + (uint64_t)(2 * k), accum);
                    }
                    wgmma_commit();
                    wgmma_wait_all();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bempty[bs]);     // this warp's reads of the slot are done
                    if (++bs == q.b_slots) { bs = 0; bph ^= 1; }
                }
                if (lane == 0) mbar_arrive(&aempty[as_]);
                if (++as_ == kASlots) { as_ = 0; aphs ^= 1; }
            }
            bar_sync(1, kNumEpiWarps * 32);
            acc_store(acc_tile, p.acc_ld, acc0, p.acc_cols, wg * 64);
            bar_sync(1, kNumEpiWarps * 32);
            epilogue_tile<SPEC, CW>(p, scr, acc_tile, nt, gw * kGM, th, tn, quarter, half, lane);
            bar_sync(1, kNumEpiWarps * 32);
            acc_store(acc_tile, p.acc_ld, acc1, p.acc_cols, wg * 64);
            bar_sync(1, kNumEpiWarps * 32);
            epilogue_tile<SPEC, CW>(p, scr, acc_tile, nt, gw * kGM + 1, th, tn, quarter, half, lane);
        }
    }
}

// Returns 1 when the launch was taken by this kernel, 0 when the shape is not eligible (caller uses mg_igemm.cu's path),
// < 0 / > 0 on error.
int conv3x3_group_launch(const mg_igemm_args* a, IgemmParams& p, int BN, int cw, int scratch_bytes, int spec, cudaStream_t stream) {
    // eligibility: 3x3, stride 1, pad 1, same-size output, transposed epilogue, an even number of 8-pixel tile columns,
    // and at least 16 rows
    if (!(a->KH == 3 && a->KW == 3 && a->stride == 1 && p.pad_h == 1 && p.pad_w == 1 && a->H == a->OH && a->W == a->OW && p.epi_impl == 1 &&
          a->OW >= 16 && a->OW % 16 == 0 && a->OH >= 16 && p.os == 1))
        return 0;
    const int acc_bytes = 128 * p.acc_ld * 4;
    {
        const int avail0 = 227 * 1024 - 1024 - 512 - scratch_bytes - acc_bytes - kASlots * kPatchBytes;
        if (avail0 / (p.acc_cols * 128) < 3) return 0;
    }
    Conv3Params q;
    memset(&q, 0, sizeof(q));
    p.TW = 8; p.TH = 16; p.TN = 1;
    p.tiles_w = a->OW / 8;
    p.tiles_h = (a->OH + 15) / 16;
    p.tiles_n = a->N;
    p.num_tiles = p.tiles_w * p.tiles_h * p.tiles_n * p.n_tiles;
    p.halo = 0;
    q.groups_w = p.tiles_w / kGM;
    q.num_groups = q.groups_w * p.tiles_h * p.tiles_n * p.n_tiles;
    const bool split = a->split != 0;
    q.steps_hi = (split && !p.merged) ? 18 : 9;
    q.steps_lo = 9;
    q.n_items = p.kchunks * (split ? 2 : 1);
    q.b_slot_bytes = p.acc_cols * 128;     // merged: [W_hi ; W_lo] = 2*BN rows; otherwise BN rows
    const int avail = 227 * 1024 - 1024 - 512 - scratch_bytes - acc_bytes - kASlots * kPatchBytes;
    q.b_slots = avail / q.b_slot_bytes;
    if (q.b_slots > kMaxBSlots) q.b_slots = kMaxBSlots;
    const size_t ring_bytes = (size_t)kASlots * kPatchBytes + (size_t)q.b_slots * q.b_slot_bytes;
    q.bar3_off = (int)ring_bytes;
    p.epi_off = (int)ring_bytes + 512;
    p.acc_off = p.epi_off + scratch_bytes;
    p.parts = p.merged ? 2 : (split ? 3 : 1);
    q.g = p;

    CUtensorMap tmA, tmA2, tmB;
    const int kelem = p.kelem;
    const int esz = a->a_fmt == 0 ? 4 : 2;
    const CUtensorMapDataType dt = a->a_fmt == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : a->a_fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    {
        cuuint64_t dims[4] = {(cuuint64_t)a->Cin, (cuuint64_t)a->W, (cuuint64_t)a->H, (cuuint64_t)a->N};
        cuuint64_t strides[3] = {(cuuint64_t)a->Cin * esz, (cuuint64_t)a->W * a->Cin * esz, (cuuint64_t)a->H * a->W * a->Cin * esz};
        cuuint32_t box[4] = {(cuuint32_t)kelem, (cuuint32_t)kPatchW, (cuuint32_t)kPatchH, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        int rc = encode_tensor_map(&tmA, (void*)a->in, dt, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
        rc = encode_tensor_map(&tmA2, (void*)(split ? a->in_lo : a->in), dt, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    {
        const int coutg = a->epi == MG_EPI_SPADE ? 2 * a->Cout : a->Cout;
        const cuuint64_t ktot = (cuuint64_t)9 * a->Cin * (split ? 2 : 1);
        cuuint64_t dims[2] = {ktot, (cuuint64_t)coutg};
        cuuint64_t strides[1] = {ktot * esz};
        cuuint32_t box[2] = {(cuuint32_t)kelem, (cuuint32_t)BN};
        cuuint32_t estr[2] = {1, 1};
        int rc = encode_tensor_map(&tmB, (void*)a->wpack, dt, 2, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const size_t smem_bytes = ring_bytes + 1024 + 512 + scratch_bytes + acc_bytes;
    static thread_local int attr_set_dev = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_set_dev != dev) {
        cudaError_t e = cudaSuccess;
        const void* kernels[6] = {(const void*)conv3x3_group_kernel<0, 16>, (const void*)conv3x3_group_kernel<0, 32>,
                                  (const void*)conv3x3_group_kernel<1, 16>, (const void*)conv3x3_group_kernel<1, 32>,
                                  (const void*)conv3x3_group_kernel<2, 16>, (const void*)conv3x3_group_kernel<2, 32>};
        for (int i = 0; i < 6 && e == cudaSuccess; ++i)
            e = cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return set_error((int)e, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        attr_set_dev = dev;
    }
    int grid = num_sms();
    if (a->max_ctas > 0 && a->max_ctas < grid) grid = a->max_ctas;
    if (grid > q.num_groups) grid = q.num_groups;
#define MG_LAUNCH3(S, C) conv3x3_group_kernel<S, C><<<grid, kThreads, smem_bytes, stream>>>(tmA, tmA2, tmB, q)
    if (spec == 1) { if (cw == 32) MG_LAUNCH3(1, 32); else MG_LAUNCH3(1, 16); }
    else if (spec == 2) { if (cw == 32) MG_LAUNCH3(2, 32); else MG_LAUNCH3(2, 16); }
    else { if (cw == 32) MG_LAUNCH3(0, 32); else MG_LAUNCH3(0, 16); }
#undef MG_LAUNCH3
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error((int)e, "conv3x3 launch: %s", cudaGetErrorString(e));
    return 1;
}

}  // namespace mg
