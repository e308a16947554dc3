// michigan_b200 — loss reductions of the train step (sm_90a).
//
// The reference evaluates its adversarial losses as chains of small eager ops per discriminator scale
// (models/networks/loss.py:60-78,100-140: interpolate -> 2x max_pool2d -> interpolate -> clamp -> mul -> mean;
// loss.py:163-175: 8x l1_loss), ~60 launches per iteration forward and as many backward.  Here:
//   * mg_edge_weight      the wide-edge weight map of one discriminator scale (loss.py:60-78) in one kernel;
//   * mg_loss_reduce      ALL terms of a loss evaluation (hinge terms of every scale, the eight feature-matching L1 terms)
//                         through one descriptor table: warp-shuffle + fp64 atomics into the loss slots;
//   * mg_loss_reduce_bwd  the matching gradients, one launch for every tensor in the table.
#include <cuda_runtime.h>
#include "mg_internal.h"

namespace mg {

// loss.py:60-66 get_wide_edges on the nearest-resized label + loss.py:73-78 weight = edges*wide_edge + (1-edges).
//   t[i,j]      = label[floor(i*H/h), floor(j*W/w)]                       (F.interpolate, mode nearest)
//   k = max(1, int(h*0.06)), p = k/2; pooled maps have size h+2p-k+1 (one more than h when k is even)
//   e_p[a,b]    = max_{k x k window at (a-p, b-p)} t - min_{same window} t   (out - (1 - maxpool(1 - t)))
//   edges[i,j]  = e_p[floor(i*hp/h), floor(j*wp/w)]                       (F.interpolate back to (h, w))
__global__ void edge_weight_kernel(const float* __restrict__ label, float* __restrict__ out, int N, int H, int W, int h, int w,
                                   int k, float wide_edge) {
    const int p = k / 2;
    const int hp = h + 2 * p - k + 1, wp = w + 2 * p - k + 1;
    const float sh = (float)H / (float)h, sw = (float)W / (float)w;
    const float ph = (float)hp / (float)h, pw = (float)wp / (float)w;
    const long long total = (long long)N * h * w;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(idx % w);
        const int i = (int)((idx / w) % h);
        const int n = (int)(idx / ((long long)w * h));
        int a = (int)floorf(i * ph), b = (int)floorf(j * pw);
        a = a < hp - 1 ? a : hp - 1; b = b < wp - 1 ? b : wp - 1;
        float mx = -1e30f, mn = 1e30f;
        for (int di = 0; di < k; ++di) {
            const int ti = a - p + di;
            if (ti < 0 || ti >= h) continue;
            int si = (int)floorf(ti * sh); si = si < H - 1 ? si : H - 1;
            for (int dj = 0; dj < k; ++dj) {
                const int tj = b - p + dj;
                if (tj < 0 || tj >= w) continue;
                int sj = (int)floorf(tj * sw); sj = sj < W - 1 ? sj : W - 1;
                const float v = __ldg(label + ((size_t)n * H + si) * W + sj);
                mx = fmaxf(mx, v); mn = fminf(mn, v);
            }
        }
        const float e = mx - mn;
        out[idx] = e * wide_edge + (1.f - e);
    }
}

// One term of a loss: slot[out_slot] += scale * sum_i f(a_i, b_i)
//   op 0  hinge, discriminator side: f = min(sign*a - 1, 0) * (w ? w_i : 1)     (loss.py:104-120)
//   op 1  plain sum: f = a                                                    (generator hinge: -mean(D(fake)), loss.py:123-124)
//   op 2  L1: f = |a - b|                                                     (GANFeatLoss, loss.py:170-172; b is detached)
//   op 3  squared difference: f = (a - b)^2                                   (content loss, loss.py:662-666; b is detached)
struct LossTerm {
    const float* a;
    const float* b;      // op 0: weight map (nullable); op 2: the other tensor
    float* ga;           // backward: gradient w.r.t. a (written, not accumulated); null = skip
    long long n;
    float scale, sign;
    int op, out_slot;
};

// grid.x blocks per term: terms range from 9 K (coarse logits) to 34 M elements (finest feature map) - enough blocks to saturate
// HBM on the large ones; blocks beyond a small term's size exit immediately
constexpr int kLossBlocksPerTerm = 592;

// (a - b)^2 with the square rounded before it is summed (no fused multiply-add across terms)
__device__ __forceinline__ float sq_diff(float a, float b) { const float d = a - b; return __fmul_rn(d, d); }

__global__ void __launch_bounds__(256) loss_reduce_kernel(const LossTerm* __restrict__ terms, double* __restrict__ slots) {
    const LossTerm t = terms[blockIdx.y];
    if ((long long)blockIdx.x * blockDim.x >= t.n && blockIdx.x != 0) return;      // no element of this term falls to this block
    float accf = 0.f;
    // 4 elements per thread per trip (float4 when the term is 16-byte aligned), fp32 partials per thread, fp64 across threads
    const bool vec = ((reinterpret_cast<uintptr_t>(t.a) | reinterpret_cast<uintptr_t>(t.b)) & 15) == 0;
    const long long n4 = vec ? t.n / 4 : 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(t.a) + i);
        float4 b = make_float4(1.f, 1.f, 1.f, 1.f);
        if (t.b) b = __ldg(reinterpret_cast<const float4*>(t.b) + i);
        if (t.op == 0) accf += fminf(t.sign * a.x - 1.f, 0.f) * b.x + fminf(t.sign * a.y - 1.f, 0.f) * b.y + fminf(t.sign * a.z - 1.f, 0.f) * b.z + fminf(t.sign * a.w - 1.f, 0.f) * b.w;
        else if (t.op == 1) accf += (a.x + a.y) + (a.z + a.w);
        else if (t.op == 2) accf += fabsf(a.x - b.x) + fabsf(a.y - b.y) + fabsf(a.z - b.z) + fabsf(a.w - b.w);
        else accf += sq_diff(a.x, b.x) + sq_diff(a.y, b.y) + sq_diff(a.z, b.z) + sq_diff(a.w, b.w);
    }
    for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
        const float a = __ldg(t.a + i);
        if (t.op == 0) accf += fminf(t.sign * a - 1.f, 0.f) * (t.b ? __ldg(t.b + i) : 1.f);
        else if (t.op == 1) accf += a;
        else if (t.op == 2) accf += fabsf(a - __ldg(t.b + i));
        else accf += sq_diff(a, __ldg(t.b + i));
    }
    double acc = (double)accf;
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    __shared__ double part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < 8; ++i) s += part[i];
        atomicAdd(slots + t.out_slot, s * (double)t.scale);
    }
}

// ga_i = gslot[out_slot] * scale * f'(a_i):  op 0: sign * w_i * [sign*a - 1 < 0];  op 1: 1;  op 2: sgn(a - b);  op 3: 2 (a - b)
__global__ void __launch_bounds__(256) loss_reduce_bwd_kernel(const LossTerm* __restrict__ terms, const float* __restrict__ gslots) {
    const LossTerm t = terms[blockIdx.y];
    if (!t.ga) return;
    const float g = __ldg(gslots + t.out_slot) * t.scale;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
        const float a = __ldg(t.a + i);
        float d;
        if (t.op == 0) d = (t.sign * a - 1.f < 0.f) ? t.sign * (t.b ? __ldg(t.b + i) : 1.f) : 0.f;
        else if (t.op == 1) d = 1.f;
        else if (t.op == 2) { const float df = a - __ldg(t.b + i); d = df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f); }
        else d = 2.f * (a - __ldg(t.b + i));
        t.ga[i] = g * d;
    }
}

}  // namespace mg

using namespace mg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mg_edge_weight(const float* label, float* out, int N, int H, int W, int h, int w, float wide_edge, void* stream) {
    if (!label || !out) return set_error(-1, "mg_edge_weight: null pointer");
    if (N < 1 || H < 1 || W < 1 || h < 1 || w < 1) return set_error(-2, "mg_edge_weight: bad size");
    int k = (int)((double)h * 0.06);
    if (k < 1) k = 1;
    const long long total = (long long)N * h * w;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
    edge_weight_kernel<<<blocks, 256, 0, ST(stream)>>>(label, out, N, H, W, h, w, k, wide_edge);
    return check_launch("mg_edge_weight");
}

extern "C" int mg_loss_reduce(const void* terms_dev, int n_terms, double* slots, void* stream) {
    if (!terms_dev || !slots) return set_error(-1, "mg_loss_reduce: null pointer");
    if (n_terms < 1 || n_terms > 65535) return set_error(-2, "mg_loss_reduce: bad term count %d", n_terms);
    loss_reduce_kernel<<<dim3(kLossBlocksPerTerm, n_terms), 256, 0, ST(stream)>>>(static_cast<const LossTerm*>(terms_dev), slots);
    return check_launch("mg_loss_reduce");
}

extern "C" int mg_loss_reduce_bwd(const void* terms_dev, int n_terms, const float* gslots, void* stream) {
    if (!terms_dev || !gslots) return set_error(-1, "mg_loss_reduce_bwd: null pointer");
    if (n_terms < 1 || n_terms > 65535) return set_error(-2, "mg_loss_reduce_bwd: bad term count %d", n_terms);
    loss_reduce_bwd_kernel<<<dim3(kLossBlocksPerTerm, n_terms), 256, 0, ST(stream)>>>(static_cast<const LossTerm*>(terms_dev), gslots);
    return check_launch("mg_loss_reduce_bwd");
}

extern "C" int mg_loss_term_bytes(void) { return (int)sizeof(mg::LossTerm); }
