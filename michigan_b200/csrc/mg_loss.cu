// michigan_b200 — loss reductions of the train step (sm_90a).
//
// The reference evaluates its adversarial losses as chains of small eager ops per discriminator scale
// (models/networks/loss.py:60-78,100-140: interpolate -> 2x max_pool2d -> interpolate -> clamp -> mul -> mean;
// loss.py:163-175: 8x l1_loss), ~60 launches per iteration forward and as many backward.  Here:
//   * mg_edge_weight      the wide-edge weight map of one discriminator scale (loss.py:60-78) in one kernel;
//   * mg_loss_reduce      ALL terms of a loss evaluation (the GAN terms of every scale in every gan_mode, the eight
//                         feature-matching L1 terms, masked or not, and the count-balanced Lab colour L1) through one
//                         descriptor table: warp-shuffle + fp64 atomics into the loss slots;
//   * mg_loss_reduce_bwd  the matching gradients, one launch for every tensor in the table.
#include <cuda_runtime.h>
#include "mg_internal.h"
#include "mg_lab.cuh"

namespace mg {

// torch's nearest source index (F.interpolate mode='nearest', upsample_nearest2d): floor(dst * (in / out)) in fp32, clamped to
// the last row / column.  scale = (float)in / (float)out.
__device__ __forceinline__ int nearest_src(int dst, float scale, int in) {
    const int s = (int)floorf(dst * scale);
    return s < in - 1 ? s : in - 1;
}

// label[n, 0, i', j'] of an [N,1,H,W] label read at (i, j) of its nearest resize to (h, w), sh = H / h, sw = W / w; rows of
// W contiguous floats, image n at n * ns (the hair channel of the one-hot label map is read in place, ns = C * H * W).
__device__ __forceinline__ float label_nearest(const float* __restrict__ label, long long ns, int n, int i, int j, int H, int W,
                                               float sh, float sw) {
    return __ldg(label + n * ns + (long long)nearest_src(i, sh, H) * W + nearest_src(j, sw, W));
}

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
        const int a = nearest_src(i, ph, hp), b = nearest_src(j, pw, wp);
        float mx = -1e30f, mn = 1e30f;
        for (int di = 0; di < k; ++di) {
            const int ti = a - p + di;
            if (ti < 0 || ti >= h) continue;
            for (int dj = 0; dj < k; ++dj) {
                const int tj = b - p + dj;
                if (tj < 0 || tj >= w) continue;
                const float v = label_nearest(label, (long long)H * W, n, ti, tj, H, W, sh, sw);
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
//   op 4  BCE with logits against the constant t: f = (1 - t) a + max(-a, 0) + log1p(exp(-|a|))   (gan_mode 'original', loss.py:81-84)
//   op 5  squared error against the constant t: f = (a - t)^2                 (gan_mode 'ls', loss.py:85-87)
// The masked ops read l = the [N,1,H,W] hair label at a's element through the nearest resize to (h, w) (loss.py:107, 157), and
// also add l over a's elements into slots[den_slot] (= sum(label1) * c, the caller divides):
//   op 6  weighted sum: f = a l                                               (generator hinge, --remove_background, loss.py:117)
//   op 7  masked hinge: f = min((sign*a - 1) l, 0)                            (discriminator hinge, --remove_background, 110-114)
//   op 8  masked L1: f = |a l - b l|                                          (GANFeatLoss.L1_loss_mask, loss.py:154-161;
//                                                                             VGGLoss.L1_loss_mask, loss.py:187-196)
//   op 9  masked squared difference: f = (a l - b l)^2                       (calc_content_loss, loss.py:664-677)
//   op 10 masked channel moments of a (NHWC or NCHW): for every (n, c), slots[out_slot + n*2C + c] += sum l a and
//         slots[out_slot + n*2C + C + c] += sum l a^2 (mg_in_stats' [N][2][C] layout; scale is not applied), and
//         slots[den_slot + n] += sum l over the image's PIXELS (each pixel once, not once per channel)    (calc_mean_std_mask,
//         loss.py:634-654).  Backward: b is a [N][3][C] fp32 table (mu', A, B) written by mg_style_loss_fwd's masked mode and
//         f'(a) = l (A + B (a - mu')).  The labels are binary (a channel of the one-hot label map, nearest-resized), l^2 = l.
//   op 11 count-balanced Lab L1 (LabColorLoss with balance_Lab, loss.py:490-531): a = fake, b = real, both [N,3,h,w] NCHW, n =
//         N h w PIXELS, label = the [N,1,h,w] hair mask (rows contiguous, image n at label + n * label_ns), table = E[256][256].
//         Per pixel: Lab of both images (mg_lab.cuh), ka = int(clamp(a_real + 128, 0, 255)), kb likewise from b_real,
//         w = E[ka][kb] l with 0 -> 1; f = w |a_fake - a_real| + w |b_fake - b_real| (each product rounded to fp32, the
//         per-pixel values summed in fp64).  Backward: ga (all three channels) = g w (sgn da  da/dfake + sgn db  db/dfake).
//   op 12 DoG orientation and confidence losses (L1OLoss, orient_filter not 'gabor', loss.py:320-385): a = rh = r * hair of
//         the response pass (mg_conv_thin's arg-max epilogue), idx its arg-max, maxv its batch maximum M, b = label2 [N,2,h,w]
//         (sin 2t, cos 2t of the target), label = hair [N,h,w] contiguous, n = N h w PIXELS (< 2^31).  Per pixel
//         conf = rh / M (IEEE division: exactly 1 at the maximiser), 0 where conf <= 0; (s, c) = table[0][idx], table[1][idx],
//         the caller's (sin, cos) of 2 (k pi / 32) (loss.py:345-348, formed by torch as the reference does);
//         ds = s conf hair - ls hair, dc likewise, dcf = conf hair - hair.  Six fp64 slots from out_slot:
//           [0] sum |ds| + |dc|   [1] sum |dcf|   [2] sum hair
//           [3] sum Lo (-rh / M^2), [4] sum Lc (-rh / M^2): the derivatives through M, Lo = [conf > 0] hair (sgn ds s + sgn dc c)
//               and Lc = [conf > 0] hair sgn dcf the per-pixel d/dconf of [0] and [1]
//           [5] the number of pixels with rh == M (torch splits the gradient of a max evenly among ties).
//         Backward, gslots[out_slot + 0..2] = (go, gc, share) with share = (go [3] + gc [4]) / [5] (formed by the caller):
//         ga = dL/dr = hair ((go Lo + gc Lc) / M + (rh == M ? share : 0)).
struct LossTerm {
    const float* a;
    const float* b;      // op 0: weight map (nullable); ops 2, 3, 8: the other tensor
    float* ga;           // backward: gradient w.r.t. a (written, not accumulated); null = skip
    long long n;
    float scale, sign;
    int op, out_slot;
    // appended for ops 4-8 (zero for ops 0-3)
    float target;        // ops 4, 5
    int den_slot;        // ops 6-8
    const float* label;  // ops 6-8: [N,1,H,W], rows contiguous, image n at label + n * label_ns
    long long label_ns;
    int C, h, w, H, W;   // ops 6-8: a is [N,C,h,w]; the label's spatial size
    int channels_last;   // ops 6-10: a (and b) laid out NHWC (the discriminator's permuted views, the VGG taps), else NCHW
    // appended for the accumulating backward (null for every term before it)
    const float* add;    // backward: ga = add + g f'(a) (may alias ga); null: ga = g f'(a).  No two terms of one launch may
                         // write the same ga.
    // appended for op 11 (null for every other op)
    const float* table;  // E[ka][kb], 256 x 256 fp32: the balance weight of the bins (a + 128, b + 128) of the real pixel
    // appended for op 12 (null for every other op)
    const unsigned char* idx;  // [N,h,w] arg-max filter k of each pixel (op 12's table: [2][32] fp32, sin and cos of 2 (k pi / 32))
    const float* maxv;         // the batch maximum M of a (one float)
};

// grid.x blocks per term: terms range from 9 K (coarse logits) to 34 M elements (finest feature map) - enough blocks to saturate
// HBM on the large ones; blocks beyond a small term's size exit immediately
constexpr int kLossBlocksPerTerm = 592;

// (a - b)^2 with the square rounded before it is summed (no fused multiply-add across terms)
__device__ __forceinline__ float sq_diff(float a, float b) { const float d = a - b; return __fmul_rn(d, d); }

// l of element i of a masked term (ops 6-10): a's index -> (n, y, x) in NCHW or NHWC order, then the label's nearest lookup
__device__ __forceinline__ float term_label(const LossTerm& t, long long i, float sh, float sw) {
    const long long chw = (long long)t.C * t.h * t.w;
    const int n = (int)(i / chw);
    const int r = (int)(i - n * chw);
    const int p = t.channels_last ? r / t.C : r % (t.h * t.w);
    return label_nearest(t.label, t.label_ns, n, p / t.w, p % t.w, t.H, t.W, sh, sw);
}

// channel of element i of a masked term
__device__ __forceinline__ int term_channel(const LossTerm& t, long long i) {
    return (int)(t.channels_last ? i % t.C : (i / ((long long)t.h * t.w)) % t.C);
}

// f of ops 4-9 and 13 at element i (l = the element's label for ops 6-9)
__device__ __forceinline__ float term_f(const LossTerm& t, float a, long long i, float l) {
    switch (t.op) {
    case 4: return __fmul_rn(1.f - t.target, a) + fmaxf(-a, 0.f) + log1pf(expf(-fabsf(a)));
    case 5: return sq_diff(a, t.target);
    case 6: return __fmul_rn(a, l);
    case 7: return fminf(__fmul_rn(t.sign * a - 1.f, l), 0.f);
    case 9: return sq_diff(__fmul_rn(a, l), __fmul_rn(__ldg(t.b + i), l));
    case 13: return expm1f(a) - a;
    default: return fabsf(__fmul_rn(a, l) - __fmul_rn(__ldg(t.b + i), l));
    }
}

// df/da of ops 4-10 and 13; ties as torch: the binary min gives each side half, |.| has gradient 0 at 0
__device__ __forceinline__ float term_df(const LossTerm& t, float a, long long i, float l) {
    switch (t.op) {
    case 4: {
        const float e = expf(-fabsf(a));
        const float sig = a >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
        return sig - t.target;
    }
    case 5: return 2.f * (a - t.target);
    case 6: return l;
    case 7: {
        const float m = __fmul_rn(t.sign * a - 1.f, l);
        return m < 0.f ? t.sign * l : (m == 0.f ? 0.5f * t.sign * l : 0.f);
    }
    case 9: return 2.f * (__fmul_rn(a, l) - __fmul_rn(__ldg(t.b + i), l)) * l;
    case 13: return expm1f(a);
    case 10: {
        const int n = (int)(i / ((long long)t.C * t.h * t.w)), c = term_channel(t, i);
        const float* co = t.b + (size_t)n * 3 * t.C + c;
        return l * (__ldg(co + t.C) + __ldg(co + 2 * t.C) * (a - __ldg(co)));
    }
    default: {
        const float df = __fmul_rn(a, l) - __fmul_rn(__ldg(t.b + i), l);
        return df > 0.f ? l : (df < 0.f ? -l : 0.f);
    }
    }
}

// op 10: each thread adds l a and l a^2 of its elements in fp32 runs of at most 32, carries the runs in fp64 and flushes them
// into the (n, c) slots whenever its (n, c) changes.  The grid stride (kLossBlocksPerTerm x 256 = 2^12 x 37) is a multiple of
// every VGG channel count, so an NHWC thread keeps one channel and flushes once per image.
__device__ __noinline__ void moments_term(const LossTerm& t, double* __restrict__ slots) {
    const float sh = (float)t.H / (float)t.h, sw = (float)t.W / (float)t.w;
    const long long chw = (long long)t.C * t.h * t.w, stride = (long long)gridDim.x * blockDim.x;
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    int cn = -1, cc = 0, run = 0;
    float f1 = 0.f, f2 = 0.f, fl = 0.f;
    double d1 = 0.0, d2 = 0.0, dl = 0.0;
    for (;; i += stride) {
        const bool more = i < t.n;
        const int n = more ? (int)(i / chw) : -2, c = more ? term_channel(t, i) : 0;
        if (n != cn || c != cc || run == 32) {
            d1 += (double)f1; d2 += (double)f2; dl += (double)fl;
            f1 = f2 = fl = 0.f;
            run = 0;
            if ((n != cn || c != cc) && cn >= 0) {
                double* s = slots + t.out_slot + (size_t)cn * 2 * t.C + cc;
                if (d1 != 0.0) atomicAdd(s, d1);
                if (d2 != 0.0) atomicAdd(s + t.C, d2);
                if (dl != 0.0) atomicAdd(slots + t.den_slot + cn, dl);
                d1 = d2 = dl = 0.0;
            }
            cn = n; cc = c;
        }
        if (!more) break;
        const float l = term_label(t, i, sh, sw), a = __ldg(t.a + i);
        const float la = __fmul_rn(a, l);
        f1 += la;
        f2 += __fmul_rn(la, a);
        if (c == 0) fl += l;
        ++run;
    }
}

// block-wide fp64 sum of one value per thread (256 threads); the result is valid in thread 0
__device__ __forceinline__ double block_sum(double acc, double* part) {
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int i = 0; i < 8; ++i) s += part[i];
    return s;
}

// op 11 at pixel i: the Lab of fake (t, f of its xyz) and the signs of its a, b differences to real, and the pixel's weight w
struct BalancedLabPixel {
    float t[3], f[3];
    float da, db, w;
};

__device__ __forceinline__ BalancedLabPixel balanced_lab_pixel(const LossTerm& t, long long i, long long hw) {
    const long long n = i / hw, p = i - n * hw;
    BalancedLabPixel px;
    float tr[3], fr[3];
    lab_xyz(t.a + (size_t)n * 3 * hw, (size_t)hw, (size_t)p, px.t);
    lab_xyz(t.b + (size_t)n * 3 * hw, (size_t)hw, (size_t)p, tr);
#pragma unroll
    for (int k = 0; k < 3; ++k) { px.f[k] = lab_f(px.t[k]); fr[k] = lab_f(tr[k]); }
    const float ar = 500.f * (fr[0] - fr[1]), br = 200.f * (fr[1] - fr[2]);
    px.da = 500.f * (px.f[0] - px.f[1]) - ar;
    px.db = 200.f * (px.f[1] - px.f[2]) - br;
    // loss.py:508-513: m = (b, a) + 128 clamped to [0, 255], truncated; the table is indexed [a bin][b bin]
    const int ka = (int)fminf(fmaxf(ar + 128.f, 0.f), 255.f), kb = (int)fminf(fmaxf(br + 128.f, 0.f), 255.f);
    const float w = __fmul_rn(__ldg(t.table + ka * 256 + kb), __ldg(t.label + n * t.label_ns + p));
    px.w = w == 0.f ? 1.f : w;                                        // loss.py:517
    return px;
}

// tp: the term's record in global memory (a reference to the kernel's local copy would put that copy on the stack)
__device__ __noinline__ void balanced_lab_term(const LossTerm* __restrict__ tp, double* __restrict__ slots, double* part) {
    const LossTerm t = *tp;
    const long long hw = (long long)t.h * t.w;
    double acc = 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
        const BalancedLabPixel px = balanced_lab_pixel(t, i, hw);
        acc += (double)__fmul_rn(px.w, fabsf(px.da)) + (double)__fmul_rn(px.w, fabsf(px.db));
    }
    const double s = block_sum(acc, part);
    if (threadIdx.x == 0) atomicAdd(slots + t.out_slot, s * (double)t.scale);
}

// inlined: a call would raise the whole backward kernel to 54 registers (35 inline)
__device__ __forceinline__ void balanced_lab_term_bwd(const LossTerm& t, float g) {
    const long long hw = (long long)t.h * t.w;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
        const BalancedLabPixel px = balanced_lab_pixel(t, i, hw);
        float v[3];
        lab_ab_backprop(px.t, px.f, sgn(px.da), sgn(px.db), g * px.w, v, 1);
        const long long n = i / hw, p = i - n * hw;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t k = ((size_t)n * 3 + c) * hw + p;
            t.ga[k] = t.add ? t.add[k] + v[c] : v[c];
        }
    }
}

// op 12 at pixel i (n < 2^31 pixels, checked by the caller): rh, hair, and the per-pixel d/dconf of the orientation and
// confidence sums (zero where conf <= 0); with kSums also |ds| + |dc| and |dcf|.  hair is read as label[i] (label_ns = h w).
struct DogPixel {
    float rh, h, lo, lc, fo, fc;
};

template <bool kSums>
__device__ __forceinline__ DogPixel dog_pixel(const LossTerm& t, int i, int hw, float M) {
    const int n = i / hw;
    DogPixel px;
    px.rh = __ldg(t.a + i);
    px.h = __ldg(t.label + i);
    const float q = px.rh / M;                                    // loss.py:341 (IEEE: no reciprocal)
    const bool pos = q > 0.f || q != q;                           // loss.py:342-343: conf * (1 - [conf <= 0])
    const float conf = pos ? q : 0.f;
    const int k = __ldg(t.idx + i);
    const float s = __ldg(t.table + k), c = __ldg(t.table + 32 + k);
    const float* lab = t.b + (size_t)i + (size_t)n * hw;          // label2[n, 0, p], p = i - n hw
    const float ds = __fmul_rn(__fmul_rn(s, conf), px.h) - __fmul_rn(__ldg(lab), px.h);
    const float dc = __fmul_rn(__fmul_rn(c, conf), px.h) - __fmul_rn(__ldg(lab + hw), px.h);
    const float dcf = __fmul_rn(conf, px.h) - px.h;
    px.lo = pos ? (sgn(ds) * s + sgn(dc) * c) * px.h : 0.f;
    px.lc = pos ? sgn(dcf) * px.h : 0.f;
    if (kSums) { px.fo = fabsf(ds) + fabsf(dc); px.fc = fabsf(dcf); }
    return px;
}

// tp: the term's record in global memory (as balanced_lab_term).  fp32 partials per thread, fp64 across threads.
__device__ __noinline__ void dog_orient_term(const LossTerm* __restrict__ tp, double* __restrict__ slots, double* part) {
    const LossTerm t = *tp;
    const int hw = t.h * t.w;
    const float M = __ldg(t.maxv);
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)t.n; i += gridDim.x * blockDim.x) {
        const DogPixel px = dog_pixel<true>(t, i, hw, M);
        const float dm = -(px.rh / M) / M;                        // d conf / d M before the [conf > 0] factor
        acc[0] += px.fo;
        acc[1] += px.fc;
        acc[2] += px.h;
        acc[3] += px.lo * dm;
        acc[4] += px.lc * dm;
        acc[5] += px.rh == M ? 1.f : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        if (k) __syncthreads();
        const double s = block_sum((double)acc[k], part);
        if (threadIdx.x == 0) atomicAdd(slots + t.out_slot + k, s);
    }
}

__device__ __forceinline__ void dog_orient_term_bwd(const LossTerm& t, const float* __restrict__ gslots) {
    const int hw = t.h * t.w;
    const float M = __ldg(t.maxv);
    const float go = __ldg(gslots + t.out_slot), gc = __ldg(gslots + t.out_slot + 1), share = __ldg(gslots + t.out_slot + 2);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)t.n; i += gridDim.x * blockDim.x) {
        const DogPixel px = dog_pixel<false>(t, i, hw, M);
        t.ga[i] = px.h * ((go * px.lo + gc * px.lc) / M + (px.rh == M ? share : 0.f));
    }
}

__global__ void __launch_bounds__(256) loss_reduce_kernel(const LossTerm* __restrict__ terms, double* __restrict__ slots) {
    const LossTerm t = terms[blockIdx.y];
    if ((long long)blockIdx.x * blockDim.x >= t.n && blockIdx.x != 0) return;      // no element of this term falls to this block
    __shared__ double part[8];
    float accf = 0.f;
    if (t.op == 10) {
        moments_term(t, slots);
        return;
    }
    if (t.op == 11) {
        balanced_lab_term(terms + blockIdx.y, slots, part);
        return;
    }
    if (t.op == 12) {
        dog_orient_term(terms + blockIdx.y, slots, part);
        return;
    }
    if (t.op >= 4) {
        // ops 4-9 and 13: one element per thread per trip, fp32 partials per thread, fp64 across threads
        const bool masked = t.op >= 6 && t.op <= 9;
        const float sh = masked ? (float)t.H / (float)t.h : 0.f, sw = masked ? (float)t.W / (float)t.w : 0.f;
        float accl = 0.f;
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
            const float l = masked ? term_label(t, i, sh, sw) : 0.f;
            accf += term_f(t, __ldg(t.a + i), i, l);
            accl += l;
        }
        const double s = block_sum((double)accf, part);
        if (threadIdx.x == 0) atomicAdd(slots + t.out_slot, s * (double)t.scale);
        if (!masked) return;
        __syncthreads();
        const double sl = block_sum((double)accl, part);
        if (threadIdx.x == 0) atomicAdd(slots + t.den_slot, sl);
        return;
    }
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
    const double s = block_sum((double)accf, part);
    if (threadIdx.x == 0) atomicAdd(slots + t.out_slot, s * (double)t.scale);
}

// ga_i = gslot[out_slot] * scale * f'(a_i):  op 0: sign * w_i * ([sign*a - 1 < 0] + [sign*a - 1 == 0] / 2);  op 1: 1;
// op 2: sgn(a - b);  op 3: 2 (a - b);  ops 4-10, 13: term_df;  op 11: balanced_lab_term_bwd;  op 12: dog_orient_term_bwd.  Op 0 at a tie: torch's binary min (the reference's torch.min(x - 1, 0))
// gives each side half the gradient.  The masked ops' denominators are folded into gslot by the caller.  With t.add the
// result is added to add_i (which may be ga itself: each element is read before the same thread writes it).
__global__ void __launch_bounds__(256) loss_reduce_bwd_kernel(const LossTerm* __restrict__ terms, const float* __restrict__ gslots) {
    const LossTerm t = terms[blockIdx.y];
    if (!t.ga) return;
    const float g = __ldg(gslots + t.out_slot) * t.scale;
    if (t.op == 11) {
        balanced_lab_term_bwd(t, g);
        return;
    }
    if (t.op == 12) {
        dog_orient_term_bwd(t, gslots);
        return;
    }
    if (t.op >= 4) {
        const bool masked = t.op >= 6 && t.op <= 10;
        const float sh = masked ? (float)t.H / (float)t.h : 0.f, sw = masked ? (float)t.W / (float)t.w : 0.f;
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
            const float l = masked ? term_label(t, i, sh, sw) : 0.f;
            const float v = g * term_df(t, __ldg(t.a + i), i, l);
            t.ga[i] = t.add ? t.add[i] + v : v;
        }
        return;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
        const float a = __ldg(t.a + i);
        float d;
        if (t.op == 0) {
            const float m = t.sign * a - 1.f;
            d = m < 0.f ? t.sign * (t.b ? __ldg(t.b + i) : 1.f) : (m == 0.f ? 0.5f * t.sign * (t.b ? __ldg(t.b + i) : 1.f) : 0.f);
        }
        else if (t.op == 1) d = 1.f;
        else if (t.op == 2) { const float df = a - __ldg(t.b + i); d = df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f); }
        else d = 2.f * (a - __ldg(t.b + i));
        const float v = g * d;
        t.ga[i] = t.add ? t.add[i] + v : v;
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
