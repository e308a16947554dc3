// michigan_b200 — per-pixel CIE Lab of the reference's Lab losses (sm_90a device helpers), shared by the Lab and hair-average
// kernels of mg_vgg.cu and the balanced Lab term of mg_loss.cu.
//
// loss.py:441-485: rgb = (img + 1) / 2; xyz = M rgb / rowsum(M); f(t) = t^(1/3) if t > 0.008856 else 7.787 t + 0.137931;
// a = 500 (f(X) - f(Y)), b = 200 (f(Y) - f(Z)).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace mg {

// static: every translation unit that includes this header keeps its own copy (the library is not built with -rdc)
static __constant__ float kLabM[3][3] = {{0.412453f, 0.357580f, 0.180423f}, {0.212671f, 0.715160f, 0.072169f}, {0.019334f, 0.119193f, 0.950227f}};
constexpr float kLabT = 0.008856f;

__device__ __forceinline__ void lab_xyz(const float* img, size_t plane, size_t off, float t[3]) {
    float rgb[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) rgb[c] = (img[c * plane + off] + 1.f) / 2.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        // the reference divides by the fp32 row sums of M (rgb2xyz: M_tmp.sum(dim=2))
        const float s = (kLabM[k][0] + kLabM[k][1]) + kLabM[k][2];
        t[k] = (kLabM[k][0] * rgb[0] + kLabM[k][1] * rgb[1] + kLabM[k][2] * rgb[2]) / s;
    }
}

__device__ __forceinline__ float lab_f(float t) { return t > kLabT ? powf(t, 1.f / 3.f) : 7.787f * t + 0.137931f; }
// f'(t), branch by branch: the cube-root branch is never evaluated at or below the threshold (t = 0 for a saturated pixel)
__device__ __forceinline__ float lab_df(float t, float ft) { return t > kLabT ? ft / (3.f * t) : 7.787f; }
__device__ __forceinline__ float sgn(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// Chain rule from (a, b) to the image: o[c * plane] = scale * d(ca a + cb b) / d img_c at a pixel with xyz t and f(t) = ft.
__device__ __forceinline__ void lab_ab_backprop(const float t[3], const float ft[3], float ca, float cb, float scale, float* o,
                                                size_t plane) {
    // d/d f(X), f(Y), f(Z), then through f' and the row-normalised M; d rgb / d img = 1/2
    const float dfk[3] = {500.f * ca, -500.f * ca + 200.f * cb, -200.f * cb};
    float dt[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) dt[k] = dfk[k] * lab_df(t[k], ft[k]) / ((kLabM[k][0] + kLabM[k][1]) + kLabM[k][2]);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane] = scale * 0.5f * (dt[0] * kLabM[0][c] + dt[1] * kLabM[1][c] + dt[2] * kLabM[2][c]);
}

}  // namespace mg
