/* michigan_b200 — C ABI of libmichigan_sm90.so (hand-written CUDA for sm_90a).
 *
 * This is the drop-in boundary for the MichiGAN data-parallel hot path.  The reference has no
 * native code: every entry point below replaces a group of PyTorch ops that the reference calls
 * from Python (file:line cited per function, relative to the reference repo root).  The reference-
 * side binding is a ctypes stub (see INTEGRATION.md and michigan_b200/_lib.py).
 *
 * Conventions (all functions):
 *   - plain device pointers + explicit sizes, fp32 data, activations NHWC ([N,H,W,C], C fastest);
 *   - `stream` is a cudaStream_t passed as void*; nothing synchronises the device, nothing
 *     allocates device memory; work is enqueued on `stream`;
 *   - return 0 on success, <0 for a rejected argument, >0 = cudaError_t; mg_last_error() gives the
 *     message of the calling thread's last failure;
 *   - re-entrant across host threads and devices.  Global state: a per-thread error string, a
 *     per-thread cache of TMA descriptors, a one-time driver entry-point lookup and the schedule
 *     knobs of mg_set_tuning (read once from the environment; every setting gives the same results).
 *     The what-if probes that skip work (env MG_DBG) exist only in the -DMG_PROBES build used by
 *     tools/; the product library has no switch that changes results.
 */
#ifndef MICHIGAN_B200_H
#define MICHIGAN_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define MG_ABI_VERSION 3

int mg_version(void);
const char* mg_last_error(void);
/* number of kernels this library has launched in the calling process (for bench.py's gpu_launches) */
long long mg_launch_count(void);
/* Schedule knobs ("MG_MERGE", "MG_HALO", "MG_HALO_PW", "MG_EPI_IMPL", "MG_EPI_IMPL_SPADE", "MG_EPI_CW16",
 * "MG_EPI_CW_SPADE", "MG_STAGES", "MG_THIN_GEMM", "MG_GROUP3", "MG_SEG_TMA", "MG_BN_FILL", "MG_EPI_REG"): initialised once from the
 * environment variable of the same name, changed here by tests and A/B tools.  Unknown name: -2 / -1. */
int mg_set_tuning(const char* name, int value);
int mg_get_tuning(const char* name);

/* activation codes */
#define MG_ACT_NONE 0
#define MG_ACT_RELU 1
#define MG_ACT_LRELU 2 /* LeakyReLU(0.2): architecture.py:84-85, discriminator.py:85,93 */
#define MG_ACT_TANH 3

/* epilogue kinds of the implicit-GEMM convolution */
#define MG_EPI_BIAS 0  /* y = act((acc*pscale + bias + residual) ...) (+ blend)            */
#define MG_EPI_SPADE 1 /* y = act(xhat*(1+gamma)+beta), gamma|beta = the two halves of acc */

/* Implicit-GEMM convolution on wgmma tensor cores (TF32 / fp16 / bf16 operands, fp32 accumulate).
 * Replaces nn.Conv2d / F.conv2d at: normalization.py:97-98,112-113 (mlp_gamma/mlp_beta, fused with
 * the modulation of normalization.py:116 and the LeakyReLU of architecture.py:84-85),
 * architecture.py:31-34,70-71,79 (conv_0/conv_1/conv_s), MaskGAN_networks.py:162-168 (ConvBlock
 * convs of BackgroundEncode2), partialconv2d.py:69 (PartialConv2d), discriminator.py:84-96.
 *
 *   in      : [N,H,W,Cin] fp32, Cin % 32 == 0 (operands are read as TF32: producers round with RNA)
 *   wpack   : [CoutG, KH*KW*Cin] fp32, K index = (kh*KW+kw)*Cin + ci  (see mg_pack_weight*)
 *   out     : [N,OH,OW,Cout]
 * MG_EPI_BIAS : CoutG == Cout.  y = acc*pscale[pix] + bias[c] + res[n,oh>>res_shift,ow>>res_shift,c];
 *               y = act(y); if (bf) y = bf[pix,c]*(1-hair[n,oh*ms,ow*ms]) + y*(1-back[n,oh*ms,ow*ms]);
 *               y *= pmul[pix].   (null pointers skip a term)
 * MG_EPI_SPADE: CoutG == 2*Cout, packed per N-tile as [gamma(BN/2) | beta(BN/2)].
 *               xh = x[n,oh>>x_shift,ow>>x_shift,c]*nscale[c] + nshift[c];
 *               y = act(xh*(gbias1[c] + acc_gamma) + (bbias[c] + acc_beta)),  gbias1 = 1 + bias_gamma.
 */
typedef struct mg_igemm_args {
    const float* in;
    const float* wpack;
    float* out;
    int32_t N, H, W, Cin;
    int32_t OH, OW, Cout;
    int32_t KH, KW, stride, pad;
    int32_t BN;        /* GEMM N tile (32..256, multiple of 32); 0 = choose */
    int32_t epi, act, round_out;
    const float* bias;
    const float* res;
    int32_t res_shift;
    const float* pscale;
    const float* pmul;
    const float* bf;
    const float* hair;
    const float* back;
    int32_t mask_stride, MH, MW; /* hair/back are [N,MH,MW] full-resolution masks */
    const float* x;
    int32_t x_shift;
    const float* nscale;
    const float* nshift;
    const float* gbias1;
    const float* bbias;
    int32_t max_ctas; /* 0 = one CTA per SM */
    /* data-gradient use (transposed convs): asymmetric extra padding (may be negative), and a strided
     * output window: out pixel (oh,ow) is stored at (oh*out_stride+out_off_h, ow*out_stride+out_off_w)
     * of an [N,OHF,OWF,Cout] tensor (0 = dense [N,OH,OW,Cout]); accumulate != 0: out += result. */
    int32_t pad_h_extra, pad_w_extra;
    int32_t out_stride, out_off_h, out_off_w, OHF, OWF, accumulate;
    /* operand format: a_fmt 0 = fp32 storage read as TF32; 1 = fp16, 2 = bf16 storage (in/in_lo/wpack are
     * then 16-bit arrays, Cin % 64 == 0).  split != 0: three-pass split precision A_hi*W_hi + A_lo*W_hi +
     * A_hi*W_lo with in = A_hi, in_lo = A_lo and wpack = [CoutG][tap][hi|lo][Cin] (mg_pack_weight16).
     * out_hi / out_lo: optional 16-bit copies of the result (hi = cvt(y), lo = cvt(y - hi)), fmt out16_fmt;
     * `out` may then be null.  fp16 hi is clamped to +-65504 first; lo is not, so it is +-inf where
     * |y - hi| >= 65520 (|y| above about 131008): fp16 hi/lo pairs carry |y| < 131008 only. */
    const void* in_lo;
    int32_t a_fmt, split;
    void* out_hi;
    void* out_lo;
    int32_t out16_fmt;
    float* aux_out; /* MG_EPI_SPADE: optional [N,OH,OW,Cout] fp32 copy of (1 + gamma), saved for mg_spade_bwd */
} mg_igemm_args;
int mg_conv_igemm(const mg_igemm_args* a, void* stream);

/* OIHW -> [O][kh][kw][I] repack, multiplied by *inv_sigma (device scalar, may be null), rounded to
 * TF32 (RNA).  Spectral-norm scaling W/sigma: torch SpectralNorm.compute_weight as applied at
 * architecture.py:38-42, normalization.py:28-29. */
int mg_pack_weight(const float* w_oihw, float* wpack, int O, int I, int KH, int KW,
                   const float* inv_sigma, int round_tf32, void* stream);
/* gamma/beta pair -> one [2C][9*128] operand, interleaved per N-tile of BN rows:
 * rows [t*BN, t*BN+BN/2) = gamma channels t*BN/2.., rows [t*BN+BN/2, (t+1)*BN) = beta channels. */
int mg_pack_weight_gb(const float* wg_oihw, const float* wb_oihw, float* wpack, int C, int I, int KH,
                      int KW, int BN, void* stream);
/* 16-bit operand variants (fmt 1 = fp16, 2 = bf16): out[o][tap][hi|lo][i]; lo present iff split != 0,
 * lo = cvt(w*inv_sigma - float(hi)).  The 3-pass split recovers ~16 (bf16) / ~22 (fp16) mantissa bits. */
int mg_pack_weight16(const float* w_oihw, void* out, int O, int I, int KH, int KW, const float* inv_sigma, int fmt,
                     int split, void* stream);
int mg_pack_weight_gb16(const float* wg_oihw, const float* wb_oihw, void* out, int C, int I, int KH, int KW, int BN,
                        int fmt, int split, void* stream);

/* Thin direct convolutions on CUDA cores (exact fp32): layers whose Cin is 3/4/7.
 * mode 0: zero padding; mode 1: reflection padding (MaskGAN_networks.py:120-121);
 * in [N,H,W,CinP] with CinP in {4,8} (channels zero-padded), w [KH*KW][CinP][Cout], Cout%32==0.
 * seg_resize > 0: `in` is the full-resolution [N,H*seg_resize,W*seg_resize,4] segmap and the conv
 * reads its legacy-nearest downsample (normalization.py:110) without materialising it. */
typedef struct mg_thin_args {
    const float* in;
    const float* w;
    const float* bias;
    float* out;
    int32_t N, H, W, CinP, OH, OW, Cout, KH, KW, stride, pad, pad_mode, seg_resize;
    int32_t act, round_out;
    const float* pscale;
    const float* pmul;
    /* optional 16-bit copies of the output (operands of the next tensor-core conv); out may be null */
    void* out_hi;
    void* out_lo;
    int32_t out16_fmt;
    /* arg-max epilogue: the Difference-of-Gaussians orientation response of L1OLoss (loss.py:320-340), selected by
     * argmax_idx != null (all three null for every other conv).  in = the [N,3,H,W] NCHW image in [-1,1], read as its gray
     * 0.299 R + 0.587 G + 0.144 B of (x+1)/2*255 (loss.py:357-358); w = the [17*17][32] bank (filter index fastest); CinP 3,
     * Cout 32, KH = KW = 17, stride 1, zero pad 8, OH = H, OW = W; bias, pscale, pmul, act, round_out, seg_resize and the
     * 16-bit copies unset.  Per pixel r = max_k max(conv_k, 0) in exact fp32, argmax_idx [N,H,W] uint8 = its first arg-max,
     * out [N,H,W] = r * argmax_mask[n,y,x] (fp32 product); *argmax_max (caller zeroes) = the maximum of out over the whole
     * call, folded in with an integer atomicMax on the bits of the non-negative floats (no host synchronisation). */
    void* argmax_idx;
    const float* argmax_mask;
    float* argmax_max;
} mg_thin_args;
int mg_conv_thin(const mg_thin_args* a, void* stream);
int mg_pack_weight_thin(const float* w_oihw, float* wt, int O, int I, int CinP, int KH, int KW, void* stream);
/* SPADE mlp_shared (normalization.py:92-96: Conv2d(label_nc=4, 128, 3, padding=1) + ReLU on the nearest-resized segmap,
 * normalization.py:110-111) as ONE K=128 tensor-core GEMM per 128-pixel tile: bf16 hi/lo split of the 3x3x4 patch and of the
 * weights concatenated along K.  Same mg_thin_args contract as mg_conv_thin restricted to CinP 4, 3x3, stride 1, pad 1,
 * Cout 128; a->w is the bf16 [128][128] operand written by mg_pack_weight_seg_tc. */
int mg_conv_seg_tc(const mg_thin_args* a, void* stream);
int mg_pack_weight_seg_tc(const float* w_oihw, void* wpack_bf16, int O, int I, void* stream);
/* debugging aid: clock64() totals of CTA 0 of mg_conv_seg_tc under env MG_DBG=16 */
int mg_debug_seg_prof(unsigned long long* host16);

/* conv_img: tanh(conv3x3(lrelu(x))) 64->3, NHWC in, NCHW out (generator.py:227-228). */
int mg_conv_img(const float* x, const float* w_oihw, const float* bias, float* out_nchw, int N, int H, int W,
                int Cin, int Cout, int act_in, int act_out, void* stream);
/* final PatchGAN logits: Cin->1, k4 s1 p2 (discriminator.py:96); out [N,OH,OW]. */
int mg_conv_to1(const float* x, const float* w_oihw, const float* bias, float* out, int N, int H, int W, int Cin,
                int KH, int KW, int pad, void* stream);

/* Param-free batch-norm statistics (sync_batchnorm/batchnorm.py:63-93,128-145; F.batch_norm path
 * batchnorm.py:65-68).  sums: [2*C] doubles (sum, sum of squares), accumulated (caller zeroes).   */
int mg_bn_stats(const float* x, long long P, int C, double* sums, void* stream);
/* the same pass also writes a bf16 copy of x (backward: bias gradient = channel sums of dY, and dY's bf16 operand copy for the
 * gradient GEMMs, in one read of dY) */
int mg_bn_stats_cvt16(const float* x, long long P, int C, double* sums, void* out_bf16, void* stream);
/* mean/var from (all-reduced) sums over `count` values -> nscale = rstd, nshift = -mean*rstd;
 * count <= 0: the sample count is read from sums[2*C] (the per-rank counts all-reduced together with the sums,
 * batchnorm.py:119 `sum_size`), so no host value depends on the other ranks' shard sizes.
 * running_mean/var momentum update with the unbiased variance of count*unbiased_mult samples (unbiased_mult =
 * 4^s when the normalised tensor is the 2^s nearest-upsampled view of x; pass null to skip).
 * clamp_mode 0: 1/sqrt(var+eps) (batchnorm.py:65-68); 1: clamp(var,eps)^-0.5 (batchnorm.py:145). */
int mg_bn_finalize(const double* sums, int C, double count, double unbiased_mult, float eps, float momentum,
                   int clamp_mode, float* nscale, float* nshift, float* running_mean, float* running_var,
                   float* mean_out, float* var_out, void* stream);
/* eval mode: nscale/nshift from running stats. */
int mg_bn_from_running(const float* running_mean, const float* running_var, int C, float eps, float* nscale,
                       float* nshift, void* stream);

/* InstanceNorm2d(affine=False) + LeakyReLU (normalization.py:47-48,52; encoder.py:173-204):
 * stats per (n,c) over HW (biased var, eps), then y = act((x-mean)*rstd) * pmul[pix]. */
int mg_in_stats(const float* x, int N, long long HW, int C, double* sums /* [N][2][C] */, void* stream);
/* ss: [N][2][C] float workspace that receives (rstd, -mean*rstd) */
int mg_in_apply(const float* x, const double* sums, float* ss, float* y, int N, long long HW, int C, float eps, int act,
                int round_out, const float* pmul, void* y_hi, void* y_lo, int out16_fmt, void* stream);

/* Input preparation (generator.py:129-142; pix2pix_model.py:549-566).
 * seg4 [N,H,W,4] = (tag0, tag1, sin(2th)*hair, cos(2th)*hair), th = orient/255*pi; orient_c==2 passes
 * the two orientation channels through (--use_ig). */
int mg_prep_seg(const float* tag_nchw, const float* orient_nchw, int orient_c, float* seg4, int N, int H, int W,
                void* stream);
/* D input [N,H,W,8] = (tag0, tag1, o0, o1, r, g, b, 0) from NHWC seg4 + NCHW image. */
int mg_prep_dinput(const float* seg4, const float* img_nchw, float* out8, int N, int H, int W, void* stream);
/* background-encoder input (encoder.py:321): img*back + noise*(1-back) -> [N,H,W,4]. */
int mg_prep_bginput(const float* img_nchw, const float* noise_nchw, const float* back, float* out4, int N, int H,
                    int W, void* stream);
/* NCHW [N,C,H,W] -> NHWC with channel padding to CP; optional per-pixel multiplier pmul [N,H,W]
 * (the `input * mask` of partialconv2d.py:69). */
int mg_nchw_to_nhwc(const float* in, float* out, int N, int C, int H, int W, int CP, const float* pmul, void* stream);
int mg_nhwc_to_nchw(const float* in, float* out, int N, int C, int H, int W, int CP, void* stream);
/* max_pool2d(k, stride 1, pad k/2) on a 1-channel map (encoder.py:296,310-313); out = 1 - pool if invert. */
int mg_maxpool_mask(const float* in, float* out, float* tmp, int N, int H, int W, int k, int invert, void* stream);
/* avg_pool2d(k3,s2,p1,count_include_pad=False) on NHWC (discriminator.py:46-49). */
int mg_avgpool3s2(const float* in, float* out, int N, int H, int W, int C, int OH, int OW, void* stream);

/* PartialConv2d mask update (partialconv2d.py:57-66): mask [N,H,W] -> ratio, update [N,OH,OW]. */
int mg_partial_mask(const float* mask, float* ratio, float* update, int N, int H, int W, int k, int stride, int pad,
                    void* stream);
/* ImageEncoder3 / ImageEncoder2 instance-wise average pooling (encoder.py:142-151, 207-220); masks are [N,MH,MW] full-res,
   MH, MW multiples of h, w.  mref == NULL: the plain spatial mean (denominator h*w: --ref_global_pool, AdaptiveAvgPool2d(1));
   mtag == NULL: broadcast with weight 1.  MH, MW are read only when a mask is given.  The backward takes the same modes. */
int mg_masked_mean_bcast(const float* x, const float* mref, const float* mtag, float* out, int N, int h, int w, int C,
                         int MH, int MW, void* stream);
/* F.interpolate(bilinear, align_corners=False) on NHWC (encoder.py:222-223). */
int mg_resize_bilinear(const float* in, float* out, int N, int H, int W, int C, int OH, int OW, void* stream);
/* nn.ReflectionPad2d(pad) on NHWC (MaskGAN_networks.py:120-121), optional TF32 (RNA) rounding. */
int mg_reflect_pad(const float* in, float* out, int N, int H, int W, int C, int pad, int round_tf32, void* out_hi,
                   void* out_lo, int out16_fmt, void* stream);

/* Spectral norm for all SN convs of a network in three launches (torch SpectralNorm.compute_weight
 * as applied at architecture.py:38-42, normalization.py:28-29).  `descs` is a DEVICE array of
 * mg_sn_desc.  training != 0: one in-place power iteration (v = normalize(W^T u), u = normalize(W v),
 * eps 1e-12) then inv_sigma = 1/(u^T W v); training == 0: inv_sigma from the stored u, v.
 * The `t` workspace must be zero on entry and is left zeroed. */
typedef struct mg_sn_desc {
    const float* w;   /* [O][K] weight_orig viewed as a matrix */
    float* u;         /* [O] weight_u */
    float* v;         /* [K] weight_v */
    float* t;         /* [K] workspace */
    float* s;         /* [O] workspace */
    float* inv_sigma; /* [1] */
    int32_t O, K;
} mg_sn_desc;
int mg_spectral_norm_batched(const void* descs, int n_layers, int max_O, int max_K, int training, float eps,
                             void* stream);

/* Weight gradient of the implicit-GEMM convs on tensor cores (TF32, MN-major operands, split-K over
 * pixels): dw[co][(kh*KW+kw)*Cin+ci] = sum_pix dy[pix,co] * x[pix*stride - pad + (kh,kw), ci].
 * dy [N,OH,OW,Cout], x [N,H,W,Cin] NHWC; dw has the packed layout of mg_pack_weight (autograd of
 * nn.Conv2d at the call sites listed for mg_conv_igemm). */
int mg_conv_wgrad(const float* dy, const float* x, float* dw, int N, int H, int W, int Cin, int OH, int OW, int Cout,
                  int KH, int KW, int stride, int pad, void* stream);
/* the same with bf16 operands (dy [N,OH,OW,Cout] and x [N,H,W,Cin] bf16; channels % 64 == 0), fp32 accumulation and output */
int mg_conv_wgrad16(const void* dy16, const void* x16, float* dw_packed, int N, int H, int W, int Cin, int OH, int OW, int Cout, int KH, int KW,
                    int stride, int pad, void* stream);

/* Operand for the data gradient (transposed conv) of a conv with weight w [O,I,KH,KW]: sub-kernel
 * taps kh = k0h + stride*j (j < Jh), flipped and transposed to [I][Jh*Jw*O], times *inv_sigma, TF32. */
int mg_pack_weight_dgrad(const float* w_oihw, float* out, int O, int I, int KH, int KW, int stride, int k0h, int Jh,
                         int k0w, int Jw, const float* inv_sigma, void* stream);
/* fp32 -> 16-bit copy (fmt 1 = fp16, 2 = bf16, round to nearest): operands of the 16-bit gradient GEMMs. */
int mg_cvt16(const float* src, void* dst, long long n, int fmt, void* stream);
/* packed [O][KH*KW*I] weight gradient -> OIHW (accumulate != 0: +=). */
int mg_unpack_wgrad(const float* dw_packed, float* dw_oihw, int O, int I, int KH, int KW, int accumulate, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Backward pass (autograd of the modules listed above; identities in SURVEY.md Appendix B).
 * ------------------------------------------------------------------------------------------- */
/* SPADE elementwise backward.  dh, h (forward output, for act'), g1 = 1+gamma (saved by the forward):
 * [N,H,W,C]; x: [N,H>>x_shift,W>>x_shift,C].  Writes dgb [N,H,W,2C] = (dgamma|dbeta) in the packed row
 * order of the forward gamma|beta operand (TF32-rounded: operand of the two gradient GEMMs), dxhat
 * [N,H,W,C], and adds sum(dxhat), sum(dxhat*xhat) to sums [2*C] doubles (normalization.py:116 + BN). */
int mg_spade_bwd(const float* dh, const float* h, const float* g1, const float* x, int x_shift, int N, int H, int W, int C,
                 const float* nscale, const float* nshift, int act, int BN, float* dgb, float* dxhat, double* sums, void* dgb16,
                 double* bias_sums, void* stream);
/* (dgb16 != null: dgb is written as bf16 [N,H,W,2C] instead - the operand of the gamma|beta gradient GEMMs, its only consumers;
 *  bias_sums != null: [2*C] doubles += per-channel sums of dgamma | dbeta = the mlp_gamma / mlp_beta bias gradients.) */
/* dx[N,hs,ws,C] (+)= nscale * sum over the 2^x_shift x 2^x_shift children of (g - m1 - xhat*m2), m = sums/count
 * (batch-norm backward through a folded nearest upsample); count <= 0: read from sums[2*C] as in mg_bn_finalize;
 * sums == null: plain child sum (upsample backward). */
int mg_bn_bwd_apply(const float* g, const float* x, int x_shift, int N, int hs, int ws, int C, const float* nscale,
                    const float* nshift, const double* sums, double count, float* dx, int accumulate, void* stream);
/* background blend backward (generator.py:186): dy = dout*(1-back), dbf (+)= dout*(1-hair). */
int mg_blend_bwd(const float* dout, const float* hair, const float* back, int N, int H, int W, int C, int mask_stride, int MH,
                 int MW, float* dy, float* dbf, int accumulate_bf, void* stream);
/* dz = dy * act'(y) * pm1[pix] * pm2[pix] (y = forward output; null pointers skip a factor). */
int mg_act_bwd(const float* dy, const float* y, float* dz, long long P, int C, int act, const float* pm1, const float* pm2,
               int round_tf32, void* stream);
/* InstanceNorm(+act,+mask) backward; ss = (rstd, shift) from mg_in_apply, sums [N][2][C] double workspace. */
int mg_in_bwd(const float* df, const float* x, const float* ss, double* sums, float* dx, int N, long long HW, int C, int act,
              const float* pmul, int round_tf32, void* stream);
/* thin conv gradients: dwt [KH*KW][CinP][Cout] (zeroed here); dimg_nchw [N,3,H,W] += data gradient of input
 * channels [c_lo, c_lo+3) (the generated image inside the discriminator input). */
int mg_thin_wgrad(const float* x, const float* dz, float* dwt, int N, int H, int W, int CinP, int OH, int OW, int Cout, int KH,
                  int KW, int stride, int pad, int pad_mode, int seg_resize, const float* relu_src, double* bias_sums, void* stream);
/* (relu_src != null: dz is first multiplied by [relu_src > 0] - the ReLU backward of SPADE's mlp_shared fused in;
 *  bias_sums != null: [Cout] doubles += per-channel sums of that dz = the conv's bias gradient; both save a full pass over dz.) */
int mg_thin_dgrad3(const float* dz, const float* wt, float* dimg_nchw, int N, int H, int W, int CinP, int OH, int OW, int Cout,
                   int KH, int KW, int stride, int pad, int c_lo, void* stream);
/* conv_img backward: dx [N,H,W,Cin] is written; dw [Cout,Cin,3,3] and db [Cout] are ACCUMULATED (zero them first).
 * Cin must divide 256 and be <= 128 (else -2, before any launch); Cout <= 3. */
int mg_conv_img_bwd(const float* dy_nchw, const float* y_nchw, const float* x, const float* w, float* dz4_ws, float* dx,
                    float* dw, float* db, int N, int H, int W, int Cin, int Cout, int act_in, int act_out, void* stream);
int mg_conv_to1_bwd(const float* dl, const float* x, const float* w, float* dx, float* dw, float* db, int N, int H, int W,
                    int Cin, int KH, int KW, int pad, int accumulate_dx, void* stream);
int mg_avgpool3s2_bwd(const float* dout, float* din_accum, int N, int H, int W, int C, int OH, int OW, void* stream);
int mg_reflect_pad_bwd(const float* dpad, float* dx, int N, int H, int W, int C, int pad, int accumulate, void* stream);
int mg_resize_bilinear_bwd(const float* dout, float* din_zeroed, int N, int H, int W, int C, int OH, int OW, void* stream);
int mg_masked_mean_bcast_bwd(const float* dout, const float* mref, const float* mtag, float* dx, int N, int h, int w, int C,
                             int MH, int MW, void* stream);
/* dW_orig (+)= (dWt - <dWt, W/sigma> u v^T) / sigma  (u, v constants: torch spectral_norm autograd). */
int mg_spectral_norm_bwd(const float* dwt, const float* w_orig, const float* u, const float* v, const float* inv_sigma,
                         double* dot_ws, float* dw, int O, long long K, int accumulate, void* stream);
int mg_pack_weight_dgrad_gb(const float* wg, const float* wb, float* out, int C, int I, int BN, void* stream);
int mg_unpack_wgrad_gb(const float* dw_packed, float* dwg, float* dwb, int C, int I, int BN, int accumulate, void* stream);

/* ---- self-attention of the InpaintGenerator (generator.py:467-485) --------------------------------------------------------
 * softmax(Q K^T) V runs as two mg_conv_igemm launches per image (1x1 convs whose weight operand is that image's K resp. V^T)
 * with this row softmax in between: x [rows, cols] scores -> probabilities, written as the operand of the second product:
 * out32 (optionally TF32-rounded) and / or 16-bit hi (+ lo residual), fmt 1 = fp16, 2 = bf16; any of them may be null. */
int mg_softmax_rows(const float* x, long long rows, int cols, float* out32, void* out_hi, void* out_lo, int out16_fmt, int round_out,
                    void* stream);

/* ---- input-pipeline prologue (data/base_dataset.py:335-396; per-sample CPU work of Dataset.__getitem__ in the reference) -----
 * mg_noise_pyramid: generate_noise (base_dataset.py:387-396): out[n,c,y,x] = mean over octaves l of cv2.resize(field_l, (H,W),
 *   INTER_LINEAR)[y,x,c]; fields: HOST array of `levels` device pointers, octave l = [N, H>>l, W>>l, 3] draws of N(0.5, 0.25^2).
 * mg_orient_rgb: trans_orient_to_rgb + ToTensor (base_dataset.py:363-385,107-110): orient [N,H,W] (0..255), label [N,H,W] ->
 *   [N,3,H,W] = uint8([(cos2t+1)/2, (sin2t+1)/2, 0.5] * label * 255) / 255 * label, t = orient/255*pi.
 * mg_hole_mask: generate_hole (base_dataset.py:335-361) for a batch: th_u[n] in [0.5,1.2] and idx_u[n] in [0,1) replace
 *   random.uniform / random.randint; centre = the floor(idx_u*count)-th nonzero pixel of orient_mask in row-major order. */
int mg_noise_pyramid(const float* const* fields, int levels, float* out_nchw, int N, int H, int W, void* stream);
int mg_orient_rgb(const float* orient, const float* label, float* out_nchw, int N, int H, int W, void* stream);
int mg_hole_mask(const float* mask, const float* orient_mask, const float* th_u, const float* idx_u, float* hole, int N, int H, int W,
                 void* stream);

/* ---- adversarial loss reductions (models/networks/loss.py:19-140 GANLoss, every gan_mode, 144-175 GANFeatLoss) ----------
 * mg_edge_weight: the wide-edge weight map of one discriminator scale (loss.py:60-78): label [N,H,W] (hair mask, 0/1)
 * -> out [N,h,w] = edges*wide_edge + (1-edges), edges = nearest-resized (maxpool_k - minpool_k) of the nearest-resized
 * label, k = max(1, int(0.06*h)), pad k/2 (pooled maps are h+1 wide for even k, resized back as the reference does). */
int mg_edge_weight(const float* label, float* out, int N, int H, int W, int h, int w, float wide_edge, void* stream);
/* One launch for all terms of a loss evaluation.  terms_dev: device array of n_terms records of mg_loss_term_bytes()
 * bytes each, layout {const float* a; const float* b; float* ga; long long n; float scale, sign; int op, out_slot;
 * float target; int den_slot; const float* label; long long label_ns; int C, h, w, H, W, channels_last; const float* add;
 * const float* table; const unsigned char* idx; const float* maxv;}:
 *   slots[out_slot] += scale * sum_i f(a_i, b_i)   (fp64 accumulation; caller zeroes `slots`)
 *   op 0: f = min(sign*a - 1, 0) * (b ? b_i : 1)   hinge, discriminator side (b = weight map)     loss.py:104-120
 *   op 1: f = a                                    generator hinge -mean(D(fake)), gan_mode 'w'     loss.py:123-124
 *   op 2: f = |a - b|                              feature matching, b detached                    loss.py:170-172
 *   op 3: f = (a - b)^2                            content loss (MSE of relu5_1), b detached       loss.py:662-666
 *   op 4: f = BCE-with-logits(a, target)           gan_mode 'original'                              loss.py:81-84
 *   op 5: f = (a - target)^2                       gan_mode 'ls'                                   loss.py:85-87
 * ops 6-10 (--remove_background) read l = label[n, 0] at a's element [n, c, y, x] (a is [N,C,h,w], NCHW or, channels_last,
 * NHWC) through the nearest resize of the [N,1,H,W] label to (h, w); ops 6-9 add l over a's elements into slots[den_slot]:
 *   op 6: f = a l                                  generator hinge                                  loss.py:117
 *   op 7: f = min((sign*a - 1) l, 0)               discriminator hinge                              loss.py:110-114
 *   op 8: f = |a l - b l|                          masked feature matching / VGG L1, b detached     loss.py:154-161, 187-196
 *   op 9: f = (a l - b l)^2                        masked content loss, b detached                  loss.py:664-677
 *   op 10: masked channel moments (calc_mean_std_mask, loss.py:634-654), l binary: per (n, c) slots[out_slot + n*2C + c] +=
 *          sum l a and slots[out_slot + n*2C + C + c] += sum l a^2 (mg_in_stats' [N][2][C] layout, fp32 runs of at most 32
 *          elements, fp64 above; scale not applied), and per image slots[den_slot + n] += sum l over its pixels (once per pixel).
 *   op 11: count-balanced Lab L1 (LabColorLoss with balance_Lab, loss.py:490-531): a = fake, b = real, both [N,3,h,w] NCHW;
 *          n = N*h*w counts PIXELS; label = the [N,1,h,w] hair mask (rows contiguous, image n at label + n*label_ns); table =
 *          E[256][256] fp32, the weight of the bins (ka, kb).  Per pixel, with the Lab of mg_lab_loss_fwd:
 *          ka = int(clamp(a_real + 128, 0, 255)), kb = int(clamp(b_real + 128, 0, 255)), w = E[ka][kb] * l, 0 -> 1;
 *          f = w |a_fake - a_real| + w |b_fake - b_real| (per-pixel fp32, summed in fp64).  ga covers all three channels:
 *          ga = add + g w (sgn da d a_fake/d fake + sgn db d b_fake/d fake), sign(0) = 0.  table is null for every other op.
 *   op 12: DoG orientation and confidence losses (L1OLoss with an orient_filter other than 'gabor', loss.py:320-385): a = rh
 *          [N,h,w] and maxv = its batch maximum M and idx = the arg-max filters, as the arg-max epilogue of mg_conv_thin wrote
 *          them; b = label2 [N,2,h,w] (sin 2t, cos 2t of the target); label = hair [N,h,w] contiguous; table = [2][32] fp32 sin
 *          and cos of 2 (k pi / 32); n = N*h*w PIXELS (< 2^31).  Per pixel conf = rh / M (IEEE division), 0 where <= 0;
 *          (s, c) = table[.][idx]; ds = s conf hair - ls hair, dc likewise, dcf = conf hair - hair.  Six slots from out_slot:
 *          sum |ds| + |dc|, sum |dcf|, sum hair, sum Lo (-rh / M^2), sum Lc (-rh / M^2), #{rh == M}, with Lo = [conf > 0] hair
 *          (sgn ds s + sgn dc c) and Lc = [conf > 0] hair sgn dcf (fp32 per thread, fp64 across threads).  M = 0 gives NaN.
 *          Backward: gslots[out_slot + 0..2] = (go, gc, share), share = (go slot3 + gc slot4) / slot5 formed by the caller;
 *          ga = dL/dr = hair ((go Lo + gc Lc) / M + [rh == M] share) (add is not applied).  idx and maxv are null for every
 *          other op.
 *   op 13: f = e^a - a - 1 (expm1f(a) - a)         the logvar half of KLDLoss, loss.py:211-213: -0.5 sum(1 + logvar -
 *          mu^2 - e^logvar) = 0.5 sum mu^2 (op 3 with b = 0) + 0.5 sum (e^logvar - logvar - 1); df/da = e^a - 1 (expm1f(a)).
 * mg_loss_reduce_bwd writes ga_i = add_i + gslots[out_slot] * scale * df/da for every term with ga != null (add null: ga_i =
 * gslots[out_slot] * scale * df/da; add may alias ga; no two terms of one launch may write the same ga).  Torch's tie rules:
 * the binary min gives each side half, |.| has gradient 0 at 0; BCE: sigmoid(a) - target.  Op 9: df/da = 2 (a l - b l) l.
 * Op 10: b is the [N][3][C] fp32 table (mu', A, B) of mg_style_loss_fwd's masked mode, df/da = l (A + B (a - mu')). */
int mg_loss_reduce(const void* terms_dev, int n_terms, double* slots, void* stream);
int mg_loss_reduce_bwd(const void* terms_dev, int n_terms, const float* gslots, void* stream);
int mg_loss_term_bytes(void);

/* ---- Gabor orientation loss (models/networks/loss.py:274-385 L1OLoss, orient_filter 'gabor'; the DoG variant is the arg-max
 * epilogue of mg_conv_thin, mg_loss_reduce op 12 and mg_orient_loss_bwd with the DoG bank, weights2 = {1, 0}) -----------------
 * img [N,3,H,W] in [-1,1]; bank [17*17][32] = the 32 Gabor kernels of gabor_fn (loss.py:214-240), filter index fastest;
 * label2 [N,2,H,W] = (sin 2t, cos 2t) of the target orientation; hair [N,H,W].
 * fwd: sums[0] += sum |orient_fake*hair - label2*hair| (both channels), sums[1] += sum log(clamp(conf,.001,1))*hair,
 *      sums[2] += sum hair  (fp64, caller zeroes);  => orient_loss = sums[0] / (2*N*H*W), confidence_loss = -sums[1] / sums[2];
 *      per pixel: winning filter index and d sums[0] / d max-response, d sums[1] / d max-response.
 * bwd: dimg = d(w[0]*sums[0] + w[1]*sums[1]) / d img, weights2 = device [2] floats (the upstream gradients folded with the
 *      normalisations above). */
int mg_orient_loss_fwd(const float* img_nchw, const float* bank, const float* label2, const float* hair, unsigned char* idx, float* dmax_l1,
                       float* dmax_log, double* sums, int N, int H, int W, void* stream);
int mg_orient_loss_bwd(const float* bank, const unsigned char* idx, const float* dmax_l1, const float* dmax_log, const float* weights2,
                       float* dimg_nchw, int N, int H, int W, void* stream);

/* ---- VGG19 perceptual loss (models/networks/loss.py:178-207 VGGLoss, architecture.py:160-190 VGG19) ----------------------
 * NHWC tensors, C a multiple of 8, every pointer 16-byte aligned.  16-bit formats: 1 = fp16, 2 = bf16.
 * mg_maxpool2_nhwc: nn.MaxPool2d(2, 2) of VGG19.features[4,9,18,27] (floor mode: out [N,H/2,W/2,C]); reads exactly one of in32 /
 *   in16 (the producer conv's fp32 or 16-bit output) and writes out32 and/or out16 (the next conv's operand, round to nearest).
 *   A window's maximum is its first element in row-major order among equals; NaN propagates (torch's rule).
 * mg_maxpool2_relu_bwd: backward of ReLU -> max-pool (features[3,4], [8,9], [17,18], [26,27]) in gather form:
 *   dx = [a > 0] * ((a is its window's arg-max ? dpool : 0) + add), with the arg-max recomputed from the same saved pre-pool
 *   tensor a (a32 or a16) by the forward's rule; add (nullable, may alias dx32) is a gradient already held for a; rows /
 *   columns of an odd-sized input outside every window get [a > 0] * add.  Writes dx32 and/or dx16 (bf16, conv_dgrad's dy16).
 * mg_relu_bwd16: ReLU backward of the layers without a pool: dz = [a > 0] * (dy + add) over n elements (n % 8 == 0), add
 *   nullable and may alias dz32; writes dz32 and/or dz16 (bf16). */
int mg_maxpool2_nhwc(const float* in32, const void* in16, int in_fmt, float* out32, void* out16, int out_fmt, int N, int H, int W, int C,
                     void* stream);
int mg_maxpool2_relu_bwd(const float* dpool, const float* a32, const void* a16, int a_fmt, const float* add, float* dx32, void* dx16,
                         int N, int H, int W, int C, void* stream);
int mg_relu_bwd16(const float* dy, const float* add, const float* a32, const void* a16, int a_fmt, float* dz32, void* dz16, long long n,
                  void* stream);

/* ---- Lab colour loss (models/networks/loss.py:403-531 LabColorLoss, balance_Lab = False; balanced: mg_loss_reduce op 11) ---
 * fake, real [N,3,H,W] in [-1,1].  Per pixel: rgb = (img+1)/2, xyz = M rgb / rowsum(M) (loss.py:441-460), f(t) = t^(1/3) if
 * t > 0.008856 else 7.787 t + 0.137931, a = 500 (f(X) - f(Y)), b = 200 (f(Y) - f(Z)) (loss.py:462-485).
 * fwd: sums[0] += sum |a_fake - a_real| + |b_fake - b_real| (fp64, caller zeroes) => loss = sums[0] / (2*N*H*W) (loss.py:523).
 * bwd: dfake = gscale[0] * d sums[0] / d fake (gscale: device float = upstream gradient / (2*N*H*W)); f' is taken branch by
 *      branch (finite at t = 0), sign(0) = 0 as in nn.L1Loss. */
int mg_lab_loss_fwd(const float* fake_nchw, const float* real_nchw, double* sums, int N, int H, int W, void* stream);
int mg_lab_loss_bwd(const float* fake_nchw, const float* real_nchw, const float* gscale, float* dfake_nchw, int N, int H, int W,
                    void* stream);

/* ---- hair-average Lab loss (models/networks/loss.py:534-621 HairAvgLabLoss, balance_Lab = False) -----------------------------
 * Replaces rgb2xyz / xyz2lab of fake and real (loss.py:549-570, the same per-pixel Lab as mg_lab_loss_fwd, L = 116 f(Y) - 16 if
 * Y > 0.008856 else 903.3 Y), cal_hair_avg (loss.py:571-577) and the L1 of the a, b averages (loss.py:601-621).
 * fake, real [N,3,H,W] fp32 in [-1,1]; mask_fake, mask_real [N,1,H,W] fp32 (the tag's and the reference's hair).
 * mg_hair_avg_lab_fwd: sums [N][2][4] fp64 (written, not accumulated) = per image {sum m L, sum m a, sum m b, sum m} of fake with
 *   mask_fake, then of real with mask_real; each product rounded to fp32 first.  Partials are added in a fixed order: two runs
 *   give the same bits.  avg = sum / (sum m, 0 -> 1); loss = mean over the N x 2 values |avg_f - avg_r| of a and b.
 * mg_hair_avg_lab_bwd: dfake = mask_fake * (T[n][0] da/dfake + T[n][1] db/dfake), T[n][j] = gscale[0] / (2N) sgn(avg_f - avg_r)
 *   / cnt_f formed on the device from `sums` (gscale: device float = upstream gradient); f' branch by branch as mg_lab_loss_bwd.
 *   real is detached: there is no d real.  With balance_Lab the host forms each image's weight from `sums` and launches the
 *   backward once per image (N = 1, pointers offset to the image), gscale = upstream gradient * w[n] / N. */
int mg_hair_avg_lab_fwd(const float* fake_nchw, const float* real_nchw, const float* mask_fake, const float* mask_real, double* sums,
                        int N, int H, int W, void* stream);
int mg_hair_avg_lab_bwd(const float* fake_nchw, const float* mask_fake, const double* sums, const float* gscale, float* dfake_nchw,
                        int N, int H, int W, void* stream);

/* ---- style and content losses (models/networks/loss.py:624-711 StyleContentLoss) -------------------------------------------
 * Replaces calc_mean_std (loss.py:624-632), calc_style_loss and calc_content_loss (loss.py:662-683) over the five VGG19 taps.
 * The per-(n, c) statistics are mg_in_stats' fp64 sums ([N][2][C]: sum x, sum x^2) of each fp32 NHWC tap, one call per tap over
 * the whole fake || target batch; the content loss is op 3 of mg_loss_reduce.
 * mg_style_loss_fwd: taps_host: HOST array of n_taps (<= 8) records of mg_style_tap_bytes() bytes, layout
 *   {const double* sums_f; const double* sums_t; float* coef; long long M; int N, C; const double* cnt_f; const double* cnt_t;}
 *   (M = pixels per image, C % 4 == 0).
 *   mu = S1 / M, sigma = sqrt((S2 - S1 mu) / (M - 1) + 1e-5) (unbiased variance, as torch.var); in fp64:
 *   loss[0] += sum over taps of (sum_nc (mu_f - mu_t)^2 + (sigma_f - sigma_t)^2) / (N*C)   (caller zeroes; one block, so the
 *   sum is bit-reproducible); coef [N][3][C] (16-byte aligned) = fp32 mu_f, mu_f - mu_t, (sigma_f - sigma_t) / sigma_f.
 *   A tap with M < 2 (relu5_1 of a crop below 32) is refused with -2; the reference returns NaN there.
 *   Masked mode (--remove_background; cnt_f, cnt_t both set, null = unmasked): S1, S2 are mg_loss_reduce op 10's sums and cnt
 *   its per-image mask sums D ([N] each), the mask binary: mu = S1 / (D + eps), sigma = sqrt((S2 - mu (2 S1 - mu D)) / (D + eps)
 *   + eps), eps = 1e-5 (calc_mean_std_mask: biased, eps twice; no pixel-count refusal); coef = op 10's backward table
 *   mu_f (1 + eps / (D_f + eps)), 2 (mu_f - mu_t) / (N C (D_f + eps)), 2 (sigma_f - sigma_t) / (N C sigma_f (D_f + eps)).
 * mg_style_tap_grad: gradient w.r.t. one fake tap x [N, HW, C] (fp32 NHWC, C % 4 == 0, 16-byte aligned), g = device [2] floats
 *   (upstream gradients of the style and content losses):
 *   out = add + g[0] (2 (mu_f - mu_t) / (N C HW) + 2 (sigma_f - sigma_t) / (N C sigma_f (HW - 1)) (x - mu_f))
 *             + g[1] 2 (x - t) / (N C HW)
 *   coef null drops the style part, content_t (the detached target tap) null the content part; add nullable, may alias out.
 * ---- background and rgb L1 losses (loss.py:388-400 RGBBackgroundL1Loss, pix2pix_model.py:51,328-333 nn.L1Loss) -------------
 * fake, tag [N,3,H,W] fp32; mask [N,H,W] (input_semantics[:, 0]) broadcast over the channels, null for the rgb loss.
 * mg_pixel_l1_fwd: sums[0] += sum |m f - m t| (products rounded first; fp64, caller zeroes) => loss = sums[0] / (3*N*H*W).
 * mg_pixel_l1_bwd: dfake = (gscale[0] sign(m f - m t)) m, sign(0) = 0 (gscale: device float = upstream gradient / (3*N*H*W)). */
int mg_style_loss_fwd(const void* taps_host, int n_taps, double* loss, void* stream);
int mg_style_tap_bytes(void);
int mg_style_tap_grad(const float* x, const float* coef, const float* content_t, const float* add, float* out, const float* g, int N,
                      long long HW, int C, void* stream);
int mg_pixel_l1_fwd(const float* fake_nchw, const float* tag_nchw, const float* mask, double* sums, int N, int H, int W, void* stream);
int mg_pixel_l1_bwd(const float* fake_nchw, const float* tag_nchw, const float* mask, const float* gscale, float* dfake_nchw, int N,
                    int H, int W, void* stream);

/* ---- data-parallel exchange over NVLink peer memory --------------------------------------------------------
 * One-shot all-reduce (sum, in place) of a small fp64 vector: replaces the SyncBN master/slave message passing of
 * sync_batchnorm/comm.py:49-133 + batchnorm.py:105-126 (ReduceAddCoalesced / Broadcast of [sum | sum of squares]).
 *   data      : [n] doubles on this rank's device, n <= mg_peer_max_elems(); holds the all-rank sum afterwards
 *               (same additions in the same order on every rank => bit-identical results everywhere)
 *   peer_bufs : HOST array of `world` device pointers, entry r = rank r's exchange buffer mapped into this
 *               process (symmetric memory / CUDA IPC), each mg_peer_buffer_bytes(world) bytes, zero-initialised
 *               once; entry `rank` is the local buffer
 *   seq       : 1, 2, 3, ... the same sequence on every rank (one number per exchange)
 *   set_tail  : != 0 -> data[n-1] is replaced by `tail` before the exchange (the per-rank sample count that
 *               travels with the BN sums, batchnorm.py:119 `sum_size`)
 *   status_dev: device int, set to 1 if a peer's vector did not arrive within ~4 s (no hang)
 * One CTA; enqueued on `stream`; no host synchronisation. */
long long mg_peer_buffer_bytes(int world);
int mg_peer_max_elems(void);
int mg_peer_allreduce_f64(double* data, int n, const void* const* peer_bufs, int world, int rank, unsigned long long seq,
                          int set_tail, double tail, int* status_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif
