// michigan_b200 — orientation losses (SURVEY.md §8f row 2; reference models/networks/loss.py:274-385 L1OLoss, orient_filter
// 'gabor' and the Difference-of-Gaussians variant).
//
// The reference builds 32 17x17 Gabor kernels ON THE FLY every call (gabor_fn, loss.py:214-240), runs 32 separate
// 1 -> 1 channel conv2d launches on the gray image, concatenates, clamps, arg-maxes, and evaluates two masked reductions:
// ~150 eager launches forward.  Here:
//   forward  : one kernel - gray tile + halo in shared memory, the 32-filter bank in shared memory ([17*17][32], float4 reads
//              broadcast to the warp), 32 accumulators per pixel in registers, clamp/arg-max/tanh/sin/cos epilogue, both
//              loss sums reduced with warp shuffles + fp64 atomics; writes per pixel the winning filter index and dL/d(response);
//   backward : one gather kernel - d gray[q] = sum over the 17x17 neighbours p of g[p] * K_{idx[p]}[q - p], then the RGB
//              coefficients (loss.py:338-340, including the reference's 0.144 blue weight).
// The DoG variant (loss.py:320-349) normalises every confidence by ONE maximum over the batch, so its forward is two-pass:
//   response : dog_response_kernel (mg_conv_thin with argmax_idx set) - the same tile and accumulators, then per pixel the first
//              arg-max, r * hair and an integer atomicMax of its bits into the batch maximum M;
//   loss     : mg_loss_reduce op 12 (mg_loss.cu) - conf = r hair / M, both loss sums and the M-path sums of the backward;
//   backward : mg_loss_reduce_bwd op 12 writes dL/dr, then orient_bwd_kernel above gathers it through the DoG bank.
#include <cuda_runtime.h>
#include "mg_internal.h"

namespace mg {

constexpr int kOK = 17, kOR = 8, kOF = 32;          // kernel size, radius, filters
constexpr int kOT = 16;                             // output tile 16 x 16, 256 threads
constexpr int kOP = kOT + 2 * kOR;                  // 32: tile + halo

__device__ __forceinline__ float gray_of(const float* img, size_t plane, size_t off) {
    // loss.py:338-340: fake = (x+1)/2*255; gray = 0.299 R + 0.587 G + 0.144 B
    const float r = (img[off] + 1.f) * 0.5f * 255.f, g = (img[plane + off] + 1.f) * 0.5f * 255.f, b = (img[2 * plane + off] + 1.f) * 0.5f * 255.f;
    return 0.299f * r + 0.587f * g + 0.144f * b;
}

// The gray tile + halo of the 16 x 16 output tile at (y0, x0) of one image (im = its [3,H,W] planes), zero outside the image.
// The helpers shared by the forward kernels take the calling kernel as a template tag: an instantiation with one caller is
// inlined before it is optimised on its own, which keeps orient_fwd_kernel's code exactly as it was before the DoG kernel
// shared it.
template <int kCaller>
__device__ __forceinline__ void orient_stage_gray(const float* __restrict__ im, float* tile, int y0, int x0, int H, int W, size_t plane) {
    for (int i = threadIdx.x; i < kOP * kOP; i += 256) {
        const int ty = i / kOP, tx = i - ty * kOP;
        const int y = y0 + ty - kOR, x = x0 + tx - kOR;
        tile[ty * (kOP + 1) + tx] = (y >= 0 && y < H && x >= 0 && x < W) ? gray_of(im, plane, (size_t)y * W + x) : 0.f;
    }
}

// resTensor[res < 0] = 0; max and argmax (first maximum) over the 32 clamped responses (loss.py:308-310, 335-337)
template <int kCaller>
__device__ __forceinline__ int orient_argmax(const float (&acc)[kOF], float& mx) {
    int best = 0;
    mx = fmaxf(acc[0], 0.f);
#pragma unroll
    for (int k = 1; k < kOF; ++k) { const float v = fmaxf(acc[k], 0.f); if (v > mx) { mx = v; best = k; } }
    return best;
}

// bank: [17*17][32] (filter index fastest).  label2: [N,2,H,W] (sin 2t, cos 2t of the target orientation, un-masked).
// sums[0] += sum |fake2 - label2| over both channels; sums[1] += sum log(clamp(conf, .001, 1)) * hair; sums[2] += sum hair.
// idx_out [N,H,W] uint8 winning filter; dconf_l1 / dconf_log [N,H,W]: d(sum |..|)/d conf and d(sum log)/d conf (unscaled).
__global__ void __launch_bounds__(256) orient_fwd_kernel(const float* __restrict__ img, const float* __restrict__ bank_g,
                                                         const float* __restrict__ label2, const float* __restrict__ hair,
                                                         unsigned char* __restrict__ idx_out, float* __restrict__ dmax_l1,
                                                         float* __restrict__ dmax_log, double* __restrict__ sums, int N, int H, int W) {
    extern __shared__ float sm[];
    float* bank = sm;                        // 289 * 32
    float* tile = sm + kOK * kOK * kOF;      // 32 * 33
    const int tiles_w = (W + kOT - 1) / kOT, tiles_h = (H + kOT - 1) / kOT;
    const size_t plane = (size_t)H * W;
    for (int i = threadIdx.x; i < kOK * kOK * kOF; i += 256) bank[i] = bank_g[i];
    double s_l1 = 0.0, s_log = 0.0, s_hair = 0.0;
    for (int t = blockIdx.x; t < N * tiles_h * tiles_w; t += gridDim.x) {
        const int n = t / (tiles_h * tiles_w), r = t - n * tiles_h * tiles_w;
        const int y0 = (r / tiles_w) * kOT, x0 = (r % tiles_w) * kOT;
        const float* im = img + (size_t)n * 3 * plane;
        __syncthreads();
        orient_stage_gray<0>(im, tile, y0, x0, H, W, plane);
        __syncthreads();
        const int ly = threadIdx.x >> 4, lx = threadIdx.x & 15;
        const int y = y0 + ly, x = x0 + lx;
        float acc[kOF];
#pragma unroll
        for (int k = 0; k < kOF; ++k) acc[k] = 0.f;
        for (int i = 0; i < kOK; ++i) {
#pragma unroll
            for (int j = 0; j < kOK; ++j) {
                const float g = tile[(ly + i) * (kOP + 1) + lx + j];
                const float4* b4 = reinterpret_cast<const float4*>(bank + (i * kOK + j) * kOF);
#pragma unroll
                for (int k4 = 0; k4 < kOF / 4; ++k4) {
                    const float4 b = b4[k4];
                    acc[4 * k4] = fmaf(g, b.x, acc[4 * k4]); acc[4 * k4 + 1] = fmaf(g, b.y, acc[4 * k4 + 1]);
                    acc[4 * k4 + 2] = fmaf(g, b.z, acc[4 * k4 + 2]); acc[4 * k4 + 3] = fmaf(g, b.w, acc[4 * k4 + 3]);
                }
            }
        }
        if (y < H && x < W) {
            // confidence = (tanh(max) + 1) / 2
            float mx;
            const int best = orient_argmax<0>(acc, mx);
            const size_t pix = (size_t)n * plane + (size_t)y * W + x;
            const float hm = hair[pix];
            const float th = tanhf(mx);
            const float conf = (th + 1.f) * 0.5f;
            const float ang = 2.f * ((float)best * 3.14159265358979323846f / (float)kOF);
            const float s = sinf(ang), c = cosf(ang);
            const float ls = label2[((size_t)n * 2) * plane + (size_t)y * W + x] * hm, lc = label2[((size_t)n * 2 + 1) * plane + (size_t)y * W + x] * hm;
            const float ds = s * conf * hm - ls, dc = c * conf * hm - lc;
            s_l1 += (double)fabsf(ds) + (double)fabsf(dc);
            const float cl = fminf(fmaxf(conf, 0.001f), 1.f);
            s_log += (double)(logf(cl) * hm);
            s_hair += (double)hm;
            // d/d(max response): through conf only (the arg-max index is piecewise constant); zero where the winner was clamped
            const float dconf_dmax = mx > 0.f ? (1.f - th * th) * 0.5f : 0.f;
            const float sgs = ds > 0.f ? 1.f : (ds < 0.f ? -1.f : 0.f), sgc = dc > 0.f ? 1.f : (dc < 0.f ? -1.f : 0.f);
            idx_out[pix] = (unsigned char)best;
            dmax_l1[pix] = (sgs * s + sgc * c) * hm * dconf_dmax;
            dmax_log[pix] = (conf >= 0.001f && conf <= 1.f) ? hm / cl * dconf_dmax : 0.f;
        }
    }
    for (int off = 16; off > 0; off >>= 1) {
        s_l1 += __shfl_xor_sync(0xffffffffu, s_l1, off); s_log += __shfl_xor_sync(0xffffffffu, s_log, off); s_hair += __shfl_xor_sync(0xffffffffu, s_hair, off);
    }
    if ((threadIdx.x & 31) == 0) { atomicAdd(sums, s_l1); atomicAdd(sums + 1, s_log); atomicAdd(sums + 2, s_hair); }
}

// dimg[n,c,q] = coef_c * 255/2 * sum_p g[p] * K_{idx[p]}[q - p + 8],  g[p] = w_l1 * dmax_l1[p] + w_log[0] * dmax_log[p]
__global__ void __launch_bounds__(256) orient_bwd_kernel(const float* __restrict__ bank_g, const unsigned char* __restrict__ idx, const float* __restrict__ dmax_l1,
                                                         const float* __restrict__ dmax_log, const float* __restrict__ wts, float* __restrict__ dimg,
                                                         int N, int H, int W) {
    extern __shared__ float sm[];
    float* bank = sm;                                    // [289][32]
    float* gt = sm + kOK * kOK * kOF;                    // 32 x 33 upstream tile
    unsigned char* it = reinterpret_cast<unsigned char*>(gt + kOP * (kOP + 1));
    const int tiles_w = (W + kOT - 1) / kOT, tiles_h = (H + kOT - 1) / kOT;
    const size_t plane = (size_t)H * W;
    for (int i = threadIdx.x; i < kOK * kOK * kOF; i += 256) bank[i] = bank_g[i];
    const float w1 = wts[0], w2 = wts[1];
    for (int t = blockIdx.x; t < N * tiles_h * tiles_w; t += gridDim.x) {
        const int n = t / (tiles_h * tiles_w), r = t - n * tiles_h * tiles_w;
        const int y0 = (r / tiles_w) * kOT, x0 = (r % tiles_w) * kOT;
        __syncthreads();
        for (int i = threadIdx.x; i < kOP * kOP; i += 256) {
            const int ty = i / kOP, tx = i - ty * kOP;
            const int y = y0 + ty - kOR, x = x0 + tx - kOR;
            float g = 0.f; unsigned char k = 0;
            if (y >= 0 && y < H && x >= 0 && x < W) {
                const size_t pix = (size_t)n * plane + (size_t)y * W + x;
                g = w1 * dmax_l1[pix] + w2 * dmax_log[pix];
                k = idx[pix];
            }
            gt[ty * (kOP + 1) + tx] = g; it[ty * kOP + tx] = k;
        }
        __syncthreads();
        const int ly = threadIdx.x >> 4, lx = threadIdx.x & 15;
        const int y = y0 + ly, x = x0 + lx;
        float acc = 0.f;
        // response[p] = sum_{i,j} gray[p + (i,j) - 8] K[i][j]  =>  d gray[q] = sum_{i,j} g[q - (i,j) + 8] K_{idx}[i][j]
        for (int i = 0; i < kOK; ++i)
#pragma unroll
            for (int j = 0; j < kOK; ++j) {
                const int ty = ly + 2 * kOR - i, tx = lx + 2 * kOR - j;      // p = q - (i,j) + 8, in tile coordinates (+8)
                const float g = gt[ty * (kOP + 1) + tx];
                if (g != 0.f) acc = fmaf(g, bank[(i * kOK + j) * kOF + it[ty * kOP + tx]], acc);
            }
        if (y < H && x < W) {
            const size_t off = (size_t)y * W + x;
            float* o = dimg + (size_t)n * 3 * plane;
            const float a = acc * 127.5f;
            o[off] = 0.299f * a; o[plane + off] = 0.587f * a; o[2 * plane + off] = 0.144f * a;
        }
    }
}

// DoG response pass (loss.py:320-340): per pixel r = max_k max(conv_k, 0), idx = its first arg-max, rh = r * hair (fp32
// product, as the reference's confidenceTensor * mask), and the batch maximum of rh folded into *mbits with an integer atomicMax
// (rh >= 0, so the order of the bit patterns is the order of the values; the caller zeroes *mbits).
__global__ void __launch_bounds__(256) dog_response_kernel(const float* __restrict__ img, const float* __restrict__ bank_g,
                                                           const float* __restrict__ hair, unsigned char* __restrict__ idx_out,
                                                           float* __restrict__ rh_out, int* __restrict__ mbits, int N, int H, int W) {
    extern __shared__ float sm[];
    float* bank = sm;                        // 289 * 32
    float* tile = sm + kOK * kOK * kOF;      // 32 * 33
    const int tiles_w = (W + kOT - 1) / kOT, tiles_h = (H + kOT - 1) / kOT;
    const size_t plane = (size_t)H * W;
    for (int i = threadIdx.x; i < kOK * kOK * kOF; i += 256) bank[i] = bank_g[i];
    float m = 0.f;
    for (int t = blockIdx.x; t < N * tiles_h * tiles_w; t += gridDim.x) {
        const int n = t / (tiles_h * tiles_w), r = t - n * tiles_h * tiles_w;
        const int y0 = (r / tiles_w) * kOT, x0 = (r % tiles_w) * kOT;
        __syncthreads();
        orient_stage_gray<1>(img + (size_t)n * 3 * plane, tile, y0, x0, H, W, plane);
        __syncthreads();
        const int ly = threadIdx.x >> 4, lx = threadIdx.x & 15;
        const int y = y0 + ly, x = x0 + lx;
        // the accumulation of orient_fwd_kernel (kept in each kernel: moved into a shared function it changes the Gabor
        // kernel's register allocation)
        float acc[kOF];
#pragma unroll
        for (int k = 0; k < kOF; ++k) acc[k] = 0.f;
        for (int i = 0; i < kOK; ++i) {
#pragma unroll
            for (int j = 0; j < kOK; ++j) {
                const float g = tile[(ly + i) * (kOP + 1) + lx + j];
                const float4* b4 = reinterpret_cast<const float4*>(bank + (i * kOK + j) * kOF);
#pragma unroll
                for (int k4 = 0; k4 < kOF / 4; ++k4) {
                    const float4 b = b4[k4];
                    acc[4 * k4] = fmaf(g, b.x, acc[4 * k4]); acc[4 * k4 + 1] = fmaf(g, b.y, acc[4 * k4 + 1]);
                    acc[4 * k4 + 2] = fmaf(g, b.z, acc[4 * k4 + 2]); acc[4 * k4 + 3] = fmaf(g, b.w, acc[4 * k4 + 3]);
                }
            }
        }
        if (y < H && x < W) {
            float mx;
            const int best = orient_argmax<1>(acc, mx);
            const size_t pix = (size_t)n * plane + (size_t)y * W + x;
            const float rh = __fmul_rn(mx, hair[pix]);
            idx_out[pix] = (unsigned char)best;
            rh_out[pix] = rh;
            m = fmaxf(m, rh);
        }
    }
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(mbits, __float_as_int(m));
}

// mg_conv_thin with argmax_idx set (see the header): the geometry of the DoG bank is the only one accepted
int orient_argmax_conv(const mg_thin_args* a, cudaStream_t stream) {
    if (!a->argmax_mask || !a->argmax_max || !a->out) return set_error(-1, "mg_conv_thin: the arg-max epilogue needs out, argmax_mask and argmax_max");
    if (a->CinP != 3 || a->Cout != kOF || a->KH != kOK || a->KW != kOK || a->stride != 1 || a->pad != kOR || a->pad_mode != 0 ||
        a->OH != a->H || a->OW != a->W || a->N < 1 || a->H < 1 || a->W < 1)
        return set_error(-2, "mg_conv_thin: the arg-max epilogue takes an NCHW RGB image (CinP 3), 32 17x17 filters, stride 1, zero pad 8");
    if (a->bias || a->pscale || a->pmul || a->out_hi || a->out_lo || a->seg_resize || a->act || a->round_out)
        return set_error(-3, "mg_conv_thin: the arg-max epilogue has no bias, activation, pixel scales, rounding or 16-bit copies");
    const size_t smem = (size_t)(kOK * kOK * kOF + kOP * (kOP + 1)) * sizeof(float);
    static thread_local int attr_dev = -1;
    int dev = 0; cudaGetDevice(&dev);
    if (attr_dev != dev) {
        const cudaError_t e = cudaFuncSetAttribute(dog_response_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        if (e != cudaSuccess) return set_error((int)e, "orient attr: %s", cudaGetErrorString(e));
        attr_dev = dev;
    }
    const int tiles = a->N * ((a->H + kOT - 1) / kOT) * ((a->W + kOT - 1) / kOT);
    int grid = 4 * num_sms();
    if (grid > tiles) grid = tiles;
    dog_response_kernel<<<grid, 256, smem, stream>>>(a->in, a->w, a->argmax_mask, static_cast<unsigned char*>(a->argmax_idx), a->out,
                                                     reinterpret_cast<int*>(a->argmax_max), a->N, a->H, a->W);
    return check_launch("mg_conv_thin");
}

}  // namespace mg

using namespace mg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mg_orient_loss_fwd(const float* img_nchw, const float* bank, const float* label2, const float* hair, unsigned char* idx,
                                  float* dmax_l1, float* dmax_log, double* sums, int N, int H, int W, void* stream) {
    if (!img_nchw || !bank || !label2 || !hair || !idx || !dmax_l1 || !dmax_log || !sums) return set_error(-1, "mg_orient_loss_fwd: null pointer");
    const size_t smem = (size_t)(kOK * kOK * kOF + kOP * (kOP + 1)) * sizeof(float);
    static thread_local int attr_dev = -1;
    int dev = 0; cudaGetDevice(&dev);
    if (attr_dev != dev) {
        cudaError_t e = cudaFuncSetAttribute(orient_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(orient_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        if (e != cudaSuccess) return set_error((int)e, "orient attr: %s", cudaGetErrorString(e));
        attr_dev = dev;
    }
    const int tiles = N * ((H + kOT - 1) / kOT) * ((W + kOT - 1) / kOT);
    int grid = 4 * num_sms();
    if (grid > tiles) grid = tiles;
    orient_fwd_kernel<<<grid, 256, smem, ST(stream)>>>(img_nchw, bank, label2, hair, idx, dmax_l1, dmax_log, sums, N, H, W);
    return check_launch("mg_orient_loss_fwd");
}

extern "C" int mg_orient_loss_bwd(const float* bank, const unsigned char* idx, const float* dmax_l1, const float* dmax_log, const float* weights2,
                                  float* dimg_nchw, int N, int H, int W, void* stream) {
    if (!bank || !idx || !dmax_l1 || !dmax_log || !weights2 || !dimg_nchw) return set_error(-1, "mg_orient_loss_bwd: null pointer");
    const size_t smem = (size_t)(kOK * kOK * kOF + kOP * (kOP + 1)) * sizeof(float) + kOP * kOP;
    const int tiles = N * ((H + kOT - 1) / kOT) * ((W + kOT - 1) / kOT);
    int grid = 4 * num_sms();
    if (grid > tiles) grid = tiles;
    orient_bwd_kernel<<<grid, 256, smem, ST(stream)>>>(bank, idx, dmax_l1, dmax_log, weights2, dimg_nchw, N, H, W);
    return check_launch("mg_orient_loss_bwd");
}
