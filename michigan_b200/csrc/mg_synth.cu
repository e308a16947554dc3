// michigan_b200 — input-pipeline prologue on the GPU (SURVEY.md §8f row 3).
//
// The reference synthesises, per sample and on the CPU inside Dataset.__getitem__ (data/pix2pix_dataset.py:66-200):
//   * the background noise image: multi-octave Gaussian noise, every octave bilinearly resized to full size with
//     cv2.resize and averaged (data/base_dataset.py:387-396 generate_noise);
//   * the orientation RGB map of --use_ig: [(cos 2t + 1)/2, (sin 2t + 1)/2, 0.5] * mask, quantised to uint8 by
//     PIL and back to [0,1] by ToTensor (base_dataset.py:363-385 trans_orient_to_rgb);
//   * the random disk "hole" inside the hair mask (base_dataset.py:335-361 generate_hole).
// At multi-GPU training speeds a CPU loader cannot produce these fast enough; the kernels below produce them for
// a whole batch from device-resident label / orientation maps.  Random draws are INPUTS (Gaussian fields, uniforms), so the
// arithmetic is testable against the reference functions on identical draws.
#include <cuda_runtime.h>
#include "mg_internal.h"

namespace mg {

constexpr int kMaxOctaves = 8;
struct NoiseArgs {
    const float* field[kMaxOctaves];   // octave l: [N, H >> l, W >> l, 3] (numpy layout of np.random.normal(size=(h, w, 3)))
    int levels;
};

// cv2.resize(..., INTER_LINEAR) source coordinate: fx = (x + 0.5) * scale - 0.5, clamped to the border (replicate).
__device__ __forceinline__ void cv_coord(int x, float scale, int n, int& x0, int& x1, float& a) {
    float fx = ((float)x + 0.5f) * scale - 0.5f;
    int sx = (int)floorf(fx);
    a = fx - (float)sx;
    if (sx < 0) { sx = 0; a = 0.f; }
    if (sx >= n - 1) { sx = n - 1; a = 0.f; }
    x0 = sx;
    x1 = sx + 1 < n ? sx + 1 : n - 1;
}

__global__ void noise_pyramid_kernel(const NoiseArgs args, float* __restrict__ out, int N, int H, int W) {
    const long long total = (long long)N * H * W;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(idx % W), y = (int)((idx / W) % H), n = (int)(idx / ((long long)W * H));
        float acc[3] = {0.f, 0.f, 0.f};
        for (int l = 0; l < args.levels; ++l) {
            const int h = H >> l, w = W >> l;
            const float* f = args.field[l] + (size_t)n * h * w * 3;
            if (l == 0) {
                const float* p = f + ((size_t)y * w + x) * 3;
                acc[0] += p[0]; acc[1] += p[1]; acc[2] += p[2];
                continue;
            }
            int x0, x1, y0, y1;
            float ax, ay;
            cv_coord(x, (float)w / (float)W, w, x0, x1, ax);
            cv_coord(y, (float)h / (float)H, h, y0, y1, ay);
            const float* p00 = f + ((size_t)y0 * w + x0) * 3;
            const float* p01 = f + ((size_t)y0 * w + x1) * 3;
            const float* p10 = f + ((size_t)y1 * w + x0) * 3;
            const float* p11 = f + ((size_t)y1 * w + x1) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float top = p00[c] + (p01[c] - p00[c]) * ax;
                const float bot = p10[c] + (p11[c] - p10[c]) * ax;
                acc[c] += top + (bot - top) * ay;
            }
        }
        const float inv = 1.f / (float)args.levels;
#pragma unroll
        for (int c = 0; c < 3; ++c) out[(((size_t)n * 3 + c) * H + y) * W + x] = acc[c] * inv;    // NCHW like torch.tensor(noise).permute(2,0,1)
    }
}

// orient [N,H,W] in 0..255, label [N,H,W] in {0,1} -> out [N,3,H,W]; uint8 quantisation (np.uint8 truncates) then / 255 (ToTensor),
// then * label once more (base_dataset.py:107-110: orient_rgb_tensor * label_tag_tensor).
__global__ void orient_rgb_kernel(const float* __restrict__ orient, const float* __restrict__ label, float* __restrict__ out, int N, int H, int W) {
    const long long hw = (long long)H * W, total = (long long)N * hw;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long n = idx / hw, pix = idx - n * hw;
        const float m = label[idx];
        const double t = (double)orient[idx] / 255.0 * 3.14159265358979323846;
        const double v0 = (cos(2.0 * t) + 1.0) / 2.0 * m * 255.0, v1 = (sin(2.0 * t) + 1.0) / 2.0 * m * 255.0, v2 = 0.5 * m * 255.0;
        float* o = out + (size_t)n * 3 * hw + pix;
        o[0] = (float)((int)v0) / 255.f * m;
        o[hw] = (float)((int)v1) / 255.f * m;
        o[2 * hw] = (float)((int)v2) / 255.f * m;
    }
}

// One block per sample.  count = #nonzero(orient_mask); rr = int(int(th * count) / pi); centre = the floor(u * count)-th nonzero
// pixel in row-major order (np.where order); hole = orient_mask * [(y-cy)^2 + (x-cx)^2 < rr] + (mask - orient_mask).
__global__ void __launch_bounds__(1024) hole_mask_kernel(const float* __restrict__ mask, const float* __restrict__ omask, const float* __restrict__ th_u,
                                                         const float* __restrict__ idx_u, float* __restrict__ hole, int H, int W) {
    const int n = blockIdx.x;
    const float* om = omask + (size_t)n * H * W;
    const float* mk = mask + (size_t)n * H * W;
    float* out = hole + (size_t)n * H * W;
    __shared__ int rowcnt[2048];
    __shared__ int s_total, s_cy, s_cx, s_rr;
    for (int y = threadIdx.x; y < H; y += blockDim.x) {
        int c = 0;
        for (int x = 0; x < W; ++x) c += om[(size_t)y * W + x] != 0.f;
        rowcnt[y] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int y = 0; y < H; ++y) tot += rowcnt[y];
        s_total = tot;
        s_cy = s_cx = -1; s_rr = 0;
        if (tot > 0) {
            const int crop = (int)((double)th_u[n] * (double)tot);
            s_rr = (int)((double)crop / 3.14159265358979323846);
            int k = (int)floorf(idx_u[n] * (float)tot);
            k = k < tot - 1 ? k : tot - 1;
            int y = 0;
            while (k >= rowcnt[y]) { k -= rowcnt[y]; ++y; }
            int x = 0;
            for (; x < W; ++x) if (om[(size_t)y * W + x] != 0.f) { if (k == 0) break; --k; }
            s_cy = y; s_cx = x;
        }
    }
    __syncthreads();
    const int tot = s_total, cy = s_cy, cx = s_cx, rr = s_rr;
    for (int i = threadIdx.x; i < H * W; i += blockDim.x) {
        if (tot == 0) { out[i] = om[i]; continue; }      // generate_hole returns orient_mask itself when it is empty
        const int y = i / W, x = i - y * W;
        const float in = ((y - cy) * (y - cy) + (x - cx) * (x - cx)) < rr ? 1.f : 0.f;
        out[i] = om[i] * in + (mk[i] - om[i]);
    }
}

}  // namespace mg

using namespace mg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mg_noise_pyramid(const float* const* fields, int levels, float* out_nchw, int N, int H, int W, void* stream) {
    if (!fields || !out_nchw) return set_error(-1, "mg_noise_pyramid: null pointer");
    if (levels < 1 || levels > kMaxOctaves) return set_error(-2, "mg_noise_pyramid: 1..%d octaves", kMaxOctaves);
    NoiseArgs a;
    for (int l = 0; l < kMaxOctaves; ++l) a.field[l] = l < levels ? fields[l] : nullptr;
    for (int l = 0; l < levels; ++l)
        if (!a.field[l] || (H >> l) < 1 || (W >> l) < 1) return set_error(-3, "mg_noise_pyramid: bad octave %d", l);
    a.levels = levels;
    const long long total = (long long)N * H * W;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
    noise_pyramid_kernel<<<blocks, 256, 0, ST(stream)>>>(a, out_nchw, N, H, W);
    return check_launch("mg_noise_pyramid");
}

extern "C" int mg_orient_rgb(const float* orient, const float* label, float* out_nchw, int N, int H, int W, void* stream) {
    if (!orient || !label || !out_nchw) return set_error(-1, "mg_orient_rgb: null pointer");
    const long long total = (long long)N * H * W;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
    orient_rgb_kernel<<<blocks, 256, 0, ST(stream)>>>(orient, label, out_nchw, N, H, W);
    return check_launch("mg_orient_rgb");
}

extern "C" int mg_hole_mask(const float* mask, const float* orient_mask, const float* th_u, const float* idx_u, float* hole, int N, int H, int W,
                            void* stream) {
    if (!mask || !orient_mask || !th_u || !idx_u || !hole) return set_error(-1, "mg_hole_mask: null pointer");
    if (H > 2048) return set_error(-2, "mg_hole_mask: H <= 2048");
    hole_mask_kernel<<<N, 1024, 0, ST(stream)>>>(mask, orient_mask, th_u, idx_u, hole, H, W);
    return check_launch("mg_hole_mask");
}
