// michigan_b200 — row softmax that emits tensor-core operands (sm_90a).
//
// InpaintGenerator's SelfAttention (reference models/networks/generator.py:467-485) is softmax(Q K^T) V over the 4096
// tokens of a 64x64 map.  Both products run on the wgmma implicit-GEMM kernel as 1x1 "convolutions" whose weight operand
// is the per-image K (resp. V^T) matrix; this kernel is the piece in between: numerically stable softmax of every score row,
// written directly in the operand format of the second product (fp32 rounded to TF32, or 16-bit hi / hi+lo), so the
// probabilities are never re-read for a conversion pass.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "mg_internal.h"
#include "mg_ptx.cuh"

namespace mg {

__device__ __forceinline__ float block_reduce(float v, float* sh, bool is_max) {
    for (int off = 16; off > 0; off >>= 1) {
        const float o = __shfl_xor_sync(0xffffffffu, v, off);
        v = is_max ? fmaxf(v, o) : v + o;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    float r = is_max ? -3.0e38f : 0.f;
    for (int i = 0; i < nw; ++i) r = is_max ? fmaxf(r, sh[i]) : r + sh[i];
    return r;
}

// one block per row; cols % 4 == 0
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, int cols, float* __restrict__ out32, void* __restrict__ hi,
                                                           void* __restrict__ lo, int fmt16, int round_out) {
    __shared__ float sh[8];
    const size_t row = blockIdx.x;
    const float4* xr = reinterpret_cast<const float4*>(x + row * cols);
    const int n4 = cols >> 2;
    float m = -3.0e38f;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = __ldg(xr + i);
        m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
    m = block_reduce(m, sh, true);
    float s = 0.f;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = __ldg(xr + i);
        s += expf(v.x - m) + expf(v.y - m) + expf(v.z - m) + expf(v.w - m);
    }
    s = block_reduce(s, sh, false);
    const float inv = 1.f / s;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = __ldg(xr + i);
        float y[4] = {expf(v.x - m) * inv, expf(v.y - m) * inv, expf(v.z - m) * inv, expf(v.w - m) * inv};
        if (round_out) {
#pragma unroll
            for (int k = 0; k < 4; ++k) y[k] = round_tf32(y[k]);
        }
        const size_t eo = row * cols + (size_t)i * 4;
        if (out32) *reinterpret_cast<float4*>(out32 + eo) = make_float4(y[0], y[1], y[2], y[3]);
        if (hi) {
            uint32_t h[2], l[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float a = y[2 * k], b = y[2 * k + 1];
                if (fmt16 == 1) {
                    const __half2 h2 = __floats2half2_rn(a, b);
                    const float2 hf = __half22float2(h2);
                    const __half2 l2 = __floats2half2_rn(a - hf.x, b - hf.y);
                    h[k] = *reinterpret_cast<const uint32_t*>(&h2); l[k] = *reinterpret_cast<const uint32_t*>(&l2);
                } else {
                    const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
                    const float2 hf = __bfloat1622float2(h2);
                    const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - hf.x, b - hf.y);
                    h[k] = *reinterpret_cast<const uint32_t*>(&h2); l[k] = *reinterpret_cast<const uint32_t*>(&l2);
                }
            }
            *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(hi) + eo) = make_uint2(h[0], h[1]);
            if (lo) *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(lo) + eo) = make_uint2(l[0], l[1]);
        }
    }
}

}  // namespace mg

extern "C" int mg_softmax_rows(const float* x, long long rows, int cols, float* out32, void* out_hi, void* out_lo, int out16_fmt, int round_out,
                               void* stream) {
    using namespace mg;
    if (!x || (!out32 && !out_hi)) return set_error(-1, "mg_softmax_rows: null pointer");
    if (cols < 4 || cols % 4 != 0 || rows < 1 || rows > 2147483647LL) return set_error(-2, "mg_softmax_rows: cols %% 4 == 0, 1 <= rows < 2^31");
    if (out_hi && (out16_fmt < 1 || out16_fmt > 2)) return set_error(-3, "mg_softmax_rows: out16_fmt must be 1 or 2");
    if (out_lo && !out_hi) return set_error(-4, "mg_softmax_rows: out_lo without out_hi");
    softmax_rows_kernel<<<(unsigned)rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, cols, out32, out_hi, out_lo, out16_fmt, round_out);
    return check_launch("mg_softmax_rows");
}
