"""The two tensor-core conv kernels (igemm_tf32_kernel, mg_igemm.cu, and conv3x3_group_kernel, mg_conv3x3.cu) and their weight
packers, called directly through ops.conv_igemm / ops.pack_weight* and compared element by element with a float64 CPU reference
of the operation they compute.

Operands are fed exactly as the kernel sees them, so that the only kernel error left is the fp32 accumulation and the fp32
epilogue:
  * TF32: activations already TF32-exact; weights = rna_tf32(fp32(w * inv_sigma)) (pack_weight, round to nearest, ties away).
  * fp16 / bf16: x.to(dtype) and fp32(w * inv_sigma).to(dtype), fp16 clamped to +-65504 first (pack_weight16).
  * split precision: exactly the three products the kernel forms, A_hi W_hi + A_lo W_hi + A_hi W_lo, with
    W_lo = cvt(v - float(W_hi)); the dropped A_lo W_lo term is printed against the unsplit conv, as information only.
  * SPADE: the gamma|beta operand of pack_weight_gb / pack_weight_gb16 against two convs with wg and wb.
The packed weight operands themselves are compared bit for bit with the layout the kernels expect.

Error model.  Per element

    |got - ref| <= k * u * R_abs + tiny,      u = 2^-24,      k = k_gemm + k_epi

where R_abs is the same fp64 formula evaluated on absolute values:
  GEMM             R_g = sum |a| |w|
  plain epilogue   R   = |pm| (|om_back| (|ps| R_g + |bias| + |res|) + |om_hair| |bf|)     (+ |out0| when accumulating)
  SPADE            R   = (|x sc| + |sh|) (|g1| + R_gamma) + |bb| + R_beta
The activations are 1-Lipschitz, so R passes through them unchanged.  k_gemm = C_GEMM sqrt(K), K = the GEMM depth in products
(KH KW Cin, times 3 for split precision); k_epi = K_EPI covers the handful of fp32 operations of the epilogue.  Measured on an
H100 80GB HBM3 at a 700 W power limit (the measured maxima are given next to each constant below); every case prints its own
max |got - ref| / (u R_abs) next to its k.

Outputs that are defined bit for bit are compared bit for bit:
  * round_out: the low 13 significand bits are zero, and the output equals rna_tf32 of the same call without round_out;
  * 16-bit copies next to the fp32 output: hi = cvt(y32) (fp16: clamped to +-65504 first), lo = cvt(y32 - float(hi));
  * 16-bit-only SPADE outputs (SPEC 1 / 2): hi + lo against the reference within the format's bound, and hi / lo equal to the
    split of the generic variant's fp32 output on the same operands;
  * strided output windows and accumulation start from a random output: every element the conv does not own comes back
    bit-identical;
  * every case runs twice: the kernels have no atomics, so both runs give the same bits.

Each case also names the kernel instantiation it must run (checked with torch.profiler), and a CPU-only test checks that every
instantiation compiled into the library is the expected variant of some case, or is listed as unreachable with its reason.
"""
import os
import re
import shutil
import subprocess
import zlib

import pytest
import torch
import torch.nn.functional as F

dev = "cuda"
U = 2.0 ** -24
TINY = 1e-30
# k_gemm = C_GEMM * sqrt(K).  Measured max |got - ref| / (u R_abs sqrt(K)) over the cases with K >= 288: 0.37 (TF32 and
# bf16 split, both kernels), 0.33 fp16; the deep cases (K = 9216 TF32, 27648 bf16 split) measured 0.20 and 0.11.
C_GEMM = 1.25
# fp32 operations of the epilogue (fma, residual add, blend fma, pmul, 1 - mask, tanhf): a few roundings of values <= R.
# Measured: the K = 32 case (where the epilogue weighs most) reached 3.4 against k = 15.1; over all cases k >= 3.9x the
# measured ratio, and the largest ratios per family were 19.5 TF32 / 11.9 fp16 / 17.8 bf16 (igemm_tf32_kernel) and 6.2 /
# 13.5 / 15.3 (conv3x3_group_kernel).
K_EPI = 8.0
LRELU_SLOPE = float(torch.tensor(0.2, dtype=torch.float32))   # the kernels multiply by 0.2f

FMT = {"tf32": 0, "f16": 1, "bf16": 2}
T16 = {"f16": torch.float16, "bf16": torch.bfloat16}
KERNEL_RE = re.compile(r"(igemm_tf32_kernel|conv3x3_group_kernel)<[^<>]*>")


def _ops():
    from michigan_b200 import ops
    return ops


def _lib():
    from michigan_b200 import _lib
    return _lib


# ============================================================================================== helpers (as in the backward tests)
def rna_tf32(t):
    """cvt.rna.tf32.f32 on finite fp32 values: round the magnitude to 10 stored mantissa bits, ties away from zero."""
    return ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def d64(t):
    return t.detach().cpu().double()


def check_close(name, got, ref, rabs, k, u=U):
    """|got - ref| <= k * u * rabs + TINY for every element; returns the measured max |got - ref| / (u R_abs)."""
    got, ref, rabs = d64(got), d64(ref), d64(rabs)
    assert got.shape == ref.shape == rabs.shape, (name, got.shape, ref.shape, rabs.shape)
    assert bool(torch.isfinite(got).all()), name
    err = (got - ref).abs()
    ratio = float((err / (u * rabs + TINY)).max())
    print("%s: max |got - ref| / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > k * u * rabs + TINY
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements out of bound; max ratio %.3g > k = %g; first at %s: got %r ref %r R_abs %r"
                             % (name, int(bad.sum()), bad.numel(), ratio, k, i, float(got[i]), float(ref[i]), float(rabs[i])))
    return ratio


def check_rounded(name, got, ref, rabs, bits, k):
    """got = ref rounded to nearest at `bits` significant bits (TF32: 11) up to k*u*R_abs of accumulated error:
    |got - ref| <= ulp(ref) / 2 + k u R_abs.  Truncation (up to a whole ulp) fails this."""
    got, ref, rabs = d64(got), d64(ref), d64(rabs)
    _, e = torch.frexp(ref)
    half_ulp = torch.ldexp(torch.ones_like(ref), (e - bits - 1).to(torch.int64))
    err = (got - ref).abs()
    ratio = float(((err - half_ulp).clamp_min(0) / (U * rabs + TINY)).max())
    print("%s: max (|got - ref| - ulp/2) / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > half_ulp + k * U * rabs + TINY
    assert not bool(bad.any()), (name, int(bad.sum()), ratio, k)
    return ratio


def cvt16(v32, fmt):
    """fp32 -> 16-bit as the packers and the epilogue convert: round to nearest even, fp16 clamped to its finite range."""
    if fmt == "f16":
        v32 = v32.clamp(-65504.0, 65504.0)
    return v32.to(T16[fmt])


def split16(v32, fmt):
    """(hi, lo) = (cvt(v), cvt(v - float(hi))); lo is not clamped (see mg_igemm_args.out_lo)."""
    hi = cvt16(v32, fmt)
    return hi, (v32 - hi.float()).to(T16[fmt])


def conv64(a, w, stride, pad_h, pad_w, OH, OW):
    """Zero-padded conv in float64: a NHWC, w OIHW -> NHWC [N, OH, OW, O].  Negative padding crops the input."""
    H, W = a.shape[1], a.shape[2]
    KH, KW = w.shape[2], w.shape[3]
    pb = max(0, (OH - 1) * stride + KH - pad_h - H)
    pr = max(0, (OW - 1) * stride + KW - pad_w - W)
    y = F.conv2d(F.pad(nchw(a), (pad_w, pr, pad_h, pb)), w, stride=stride)
    return nhwc(y[:, :, :OH, :OW])


def gemm_ref(pairs, stride, pad_h, pad_w, OH, OW):
    """sum over (activation, weight) operand pairs of conv64 -> (ref, R_g)."""
    ref = sum(conv64(d64(a), d64(w), stride, pad_h, pad_w, OH, OW) for a, w in pairs)
    rabs = sum(conv64(d64(a).abs(), d64(w).abs(), stride, pad_h, pad_w, OH, OW) for a, w in pairs)
    return ref, rabs


def up(t, s, OH, OW):
    """Nearest 2^s upsample of an NHWC tensor, cropped to OH x OW."""
    f = 1 << s
    return t.repeat_interleave(f, 1).repeat_interleave(f, 2)[:, :OH, :OW] if s else t


def act64(y, act):
    if act == 1:
        return y.clamp_min(0)
    if act == 2:
        return torch.where(y > 0, y, LRELU_SLOPE * y)
    if act == 3:
        return torch.tanh(y)
    return y


def packed(w, fmt, split, inv=None):
    """Expected packed operand [O][tap][hi|lo][I] of pack_weight / pack_weight16, and the effective weights (OIHW) per part."""
    v = w * inv if inv is not None else w.clone()          # fp32 product, as the packers form it
    O, I, KH, KW = w.shape
    tap = lambda t: t.permute(0, 2, 3, 1).reshape(O, KH * KW, 1, I)
    if fmt == "tf32":
        wr = rna_tf32(v)
        return tap(wr).reshape(O, -1), [wr]
    hi, lo = split16(v, fmt)
    if not split:
        return tap(hi).reshape(O, -1), [hi]
    return torch.cat([tap(hi), tap(lo)], 2).reshape(O, -1), [hi, lo]


def packed_gb(wg, wb, fmt, split, bn):
    """Expected gamma|beta operand: per N tile of bn rows, [gamma(bn/2) | beta(bn/2)]; effective (wg, wb) parts."""
    C = wg.shape[0]
    (pg, eg), (pb, eb) = packed(wg, fmt, split), packed(wb, fmt, split)
    half = bn // 2
    out = torch.cat([pg.reshape(C // half, half, -1), pb.reshape(C // half, half, -1)], 1).reshape(2 * C, -1)
    return out, eg, eb


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _same_bits(name, a, b):
    a, b = a.cpu(), b.cpu()
    assert a.shape == b.shape and a.dtype == b.dtype, (name, a.shape, b.shape, a.dtype, b.dtype)
    neq = _bits(a) != _bits(b)
    assert not bool(neq.any()), "%s: %d elements differ, first at %s" % (name, int(neq.sum()), tuple(neq.nonzero()[0].tolist()))


# ============================================================================================== kernel variants
def IG(fmt, bn, merged, spec, cw):
    return "igemm_tf32_kernel<%d,%d,%s,%d,%d>" % (fmt, bn, str(bool(merged)).lower(), spec, cw)


def G3(fmt, bn, merged, spec, cw, reg):
    return "conv3x3_group_kernel<%d,%d,%s,%d,%d,%s>" % (fmt, bn, str(bool(merged)).lower(), spec, cw, str(bool(reg)).lower())


def _norm(name):
    return re.sub(r"\s+", "", name)


# Compiled instantiations that no launcher setting selects.  conv3x3_group_launch needs >= 3 weight slots next to the staged
# epilogue's shared memory (two 41 KB patches + the fp32 accumulator tile + the scratch); with 32-channel chunks (36 KB of scratch)
# and a 128-column accumulator tile only 2 fit, so the launcher returns "not eligible" and the per-tap kernel runs the layer
# (case cw32_group_falls_back_bn128 checks that).  They exist because the variant set is the same for both kernels.
_NO_ROOM = "CW 32 staged epilogue with a 128-column accumulator leaves < 3 weight slots: the per-tap kernel runs instead"
UNREACHABLE = {G3(f, 128, False, s, 32, False): _NO_ROOM for f in (0, 1, 2) for s in (0, 1, 2)}
UNREACHABLE.update({G3(f, 64, True, 0, 32, False): _NO_ROOM for f in (1, 2)})


# ============================================================================================== cases
def case(name, variant, **kw):
    c = dict(name=name, variant=_norm(variant), fmt="tf32", split=False, N=2, H=16, W=16, Cin=None, Cout=64, k=3, s=1, p=1,
             act=2, feats=(), knobs={}, bn=0, ctas=5, inv=None, spade=None, out16=None, want_f32=True, extra=None, out_hw=None)
    c.update(kw)
    if c["Cin"] is None:
        c["Cin"] = 32 if c["fmt"] == "tf32" else 64
    c["feats"] = set(c["feats"])
    return c


NOG3 = {"MG_GROUP3": 0}
HAND = [
    # ---- geometry: k1 / k3 / k4, stride 1 / 2, pad 0 / 1 / 2, the networks' odd sizes, non-square maps, partial row tiles
    case("k1s1p0_33x35", IG(0, 64, 0, 0, 16), H=33, W=35, k=1, p=0, feats={"bias"}, inv=0.61),
    case("k3s2p1_67x33_cout32", IG(0, 32, 0, 0, 16), H=67, W=33, Cin=64, Cout=32, s=2, act=1, feats={"bias"}, inv=1.7, ctas=3),
    case("k4s2p1_13x11_bf16_cout96", IG(2, 32, 0, 0, 16), H=13, W=11, Cout=96, k=4, s=2, act=3, feats={"bias"}, fmt="bf16"),
    case("k3s1p2_13x11_f16_cout160", IG(1, 32, 0, 0, 16), H=13, W=11, Cout=160, p=2, feats={"bias"}, fmt="f16", inv=0.37),
    case("k4s2p2_35x33", IG(0, 64, 0, 0, 16), H=35, W=33, k=4, s=2, p=2, act=0, feats={"bias", "pscale"}),
    case("group_16x48_nonsquare", G3(0, 64, 0, 0, 16, 1), W=48, feats={"bias", "res"}, inv=0.8),
    case("group_oh40_bf16split_merged", G3(2, 64, 1, 0, 16, 1), H=40, W=32, fmt="bf16", split=True, feats={"bias", "res"}, ctas=1),
    case("group_oh40_f16_bn128_staged", G3(1, 128, 0, 0, 16, 0), H=40, W=16, Cout=128, bn=128, fmt="f16", feats={"bias"},
         out16=("f16", False)),
    case("group_reg_conv1_blend2_res1", G3(2, 64, 1, 0, 16, 1), H=32, W=32, fmt="bf16", split=True,
         feats={"bias", "res1", "blend2"}, ctas=3),
    case("group_bf16split_3pass_cout256", G3(2, 128, 0, 0, 16, 0), Cout=256, bn=128, fmt="bf16", split=True, feats={"bias", "res"}),
    # ---- small maps: one tile holds several images (TN > 1); blend with mask_stride 2 / 4 and res_shift 1 (conv_1 of the
    # SPADE ResNet blocks, architecture.py:146 / generator.py:163)
    case("8x8_N3_tn2_conv1", IG(0, 32, 0, 0, 16), N=3, H=8, W=8, Cout=32, feats={"bias", "res1", "blend2"}),
    case("4x4_N5_tn8_merged", IG(2, 64, 1, 0, 16), N=5, H=4, W=4, fmt="bf16", split=True, feats={"bias", "res1", "blend4"}),
    case("2x2_N3_tn32_f16", IG(1, 32, 0, 0, 16), N=3, H=2, W=2, Cout=96, fmt="f16", feats={"bias", "res1", "blend2"}),
    case("1x1_N3_tn128_bnfill1", IG(0, 64, 0, 0, 16), N=3, H=1, W=1, Cout=256, feats={"bias", "blend4"}),
    case("1x1_N3_tn128_bnfill0", IG(0, 128, 0, 0, 16), N=3, H=1, W=1, Cout=256, feats={"bias", "blend4"},
         knobs={"MG_BN_FILL": 0}),
    case("8x8_cout256_bnfill1", IG(2, 64, 0, 0, 16), H=8, W=8, Cout=256, fmt="bf16", feats={"bias", "res"}),
    case("8x8_cout256_bnfill0", IG(2, 128, 0, 0, 16), H=8, W=8, Cout=256, fmt="bf16", feats={"bias", "res"},
         knobs={"MG_BN_FILL": 0}),
    # ---- SPADE at C = 32 (BN 64), 64, 128, 256 (BN 128); aux + round_out as in architecture.py:118 (TF32 mode)
    case("spade_c32_aux_round", G3(0, 64, 0, 0, 16, 1), W=32, spade=(32, 0), feats={"aux", "round"}),
    case("spade_c64_f16_aux_xs1", G3(1, 128, 0, 0, 16, 0), act=0, fmt="f16", spade=(64, 1), feats={"aux"}),
    case("spade_c128_spec1_bf16split", G3(2, 128, 0, 1, 16, 1), fmt="bf16", split=True, spade=(128, 0),
         out16=("bf16", True), want_f32=False),
    case("spade_c256_spec2_pertap", IG(0, 128, 0, 2, 16), H=12, W=12, act=0, spade=(256, 1), out16=("bf16", True),
         want_f32=False),
    case("spade_c32_spec1_merged_tn2", IG(2, 64, 1, 1, 16), N=3, H=8, W=8, fmt="bf16", split=True, spade=(32, 1),
         out16=("bf16", True), want_f32=False),
    # ---- epilogue terms in the combinations the networks use
    case("partial_conv_pscale_pmul", IG(0, 64, 0, 0, 16), H=34, W=34, s=2, act=0, feats={"bias", "pscale", "pmul"}),
    case("disc_k4s2_round", IG(0, 64, 0, 0, 16), Cin=64, Cout=128, H=18, W=18, k=4, s=2, p=2, feats={"bias", "round"}),
    case("disc_f16_out16_nolo", IG(1, 64, 0, 0, 16), H=10, W=10, k=4, p=2, fmt="f16", feats={"bias"}, out16=("f16", False),
         want_f32=False),
    case("lrelu_exact_zeros", IG(0, 32, 0, 0, 16), H=6, W=10, Cout=32, feats={"bias", "zero"}),
    case("f16_out16_beyond_65504_group", G3(1, 64, 0, 0, 16, 1), fmt="f16", feats={"bias", "big"}, act=0, out16=("f16", True)),
    case("f16_out16_beyond_65504_rowlane", IG(1, 64, 0, 0, 16), fmt="f16", feats={"bias", "big"}, act=0, out16=("f16", True),
         knobs={"MG_EPI_IMPL": 0}),
    case("bf16_out16_split_round", IG(0, 64, 0, 0, 16), H=12, W=20, feats={"bias", "round"}, out16=("bf16", True)),
    # ---- knobs: every schedule must give results within the same bound
    case("group3_off", IG(2, 64, 1, 0, 16), fmt="bf16", split=True, feats={"bias", "res"}, knobs=NOG3),
    case("epi_reg0_merged", G3(2, 64, 1, 0, 16, 0), fmt="bf16", split=True, feats={"bias", "blend2"}, knobs={"MG_EPI_REG": 0}),
    case("merge0_3pass_group", G3(2, 64, 0, 0, 16, 1), fmt="bf16", split=True, feats={"bias", "res1"}, knobs={"MG_MERGE": 0}),
    case("merge0_3pass_pertap", IG(1, 64, 0, 0, 16), H=12, W=12, fmt="f16", split=True, feats={"bias"}, knobs={"MG_MERGE": 0}),
    case("halo_pw10_tf32", IG(0, 64, 0, 0, 16), feats={"bias", "res"}, knobs={"MG_HALO": 1, "MG_HALO_PW": 10}),
    case("halo_pw16_bf16split_40x24", IG(2, 64, 1, 0, 16), H=40, W=24, fmt="bf16", split=True, feats={"bias", "res1", "pmul"},
         knobs={"MG_HALO": 1, "MG_HALO_PW": 16}, ctas=3),
    case("halo_spade_c32_aux", IG(1, 64, 0, 0, 16), fmt="f16", spade=(32, 1), feats={"aux"}, knobs={"MG_HALO": 1, "MG_HALO_PW": 10}),
    case("rowlane_33x35_all_terms", IG(0, 64, 0, 0, 16), H=33, W=35, feats={"bias", "res", "pscale", "pmul", "blend2"},
         knobs={"MG_EPI_IMPL": 0}, inv=0.9),
    case("rowlane_spade_c64_aux_round", IG(0, 128, 0, 0, 16), spade=(64, 1), feats={"aux", "round"},
         knobs={"MG_EPI_IMPL_SPADE": 0}),
    case("cw32_group_staged", G3(0, 64, 0, 0, 32, 0), Cout=128, bn=64, feats={"bias", "res"},
         knobs={"MG_EPI_CW16": 0, "MG_EPI_REG": 0}),
    case("cw32_group_falls_back_bn128", IG(0, 128, 0, 0, 32), Cout=128, bn=128, feats={"bias", "res"},
         knobs={"MG_EPI_CW16": 0}),
    case("cw32_spade_c64_f16", IG(1, 128, 0, 0, 32), H=12, W=12, fmt="f16", spade=(64, 0), feats={"aux"},
         knobs={"MG_EPI_CW_SPADE": 32}),
    case("stages3_bf16_k3s2", IG(2, 64, 0, 0, 16), H=33, W=35, s=2, fmt="bf16", feats={"bias"}, knobs={"MG_STAGES": 3}, ctas=3),
    case("stages3_merged_ctas1", IG(2, 64, 1, 0, 16), H=12, W=20, fmt="bf16", split=True, feats={"bias", "res"},
         knobs={"MG_STAGES": 3}, ctas=1),
    # ---- accumulation, strided output windows (conv_dgrad's parity classes, the VGG dgrad at architecture.py:338), ragged tiles
    case("window_s2_accumulate", IG(0, 64, 0, 0, 16), H=9, W=10, k=2, p=0, act=0, feats={"bias", "accumulate"},
         extra=dict(pad_h_extra=1, pad_w_extra=0, out_stride=2, out_off_h=1, out_off_w=0, OHF=19, OWF=21), out_hw=(9, 10)),
    case("window_negative_pad_bf16", IG(2, 32, 0, 0, 16), H=9, W=9, Cout=32, p=0, act=0, fmt="bf16",
         extra=dict(pad_h_extra=-1, pad_w_extra=-2, out_stride=2, out_off_h=0, out_off_w=1, OHF=16, OWF=14), out_hw=(6, 5)),
    case("window_group_offset_accumulate", G3(0, 64, 0, 0, 16, 1), p=0, act=0, feats={"accumulate"},
         extra=dict(pad_h_extra=1, pad_w_extra=1, out_stride=1, out_off_h=1, out_off_w=2, OHF=18, OWF=19), out_hw=(16, 16)),
    case("accumulate_ragged_group_oh40", G3(2, 64, 0, 0, 16, 1), H=40, fmt="bf16", act=0, feats={"bias", "accumulate"}),
    case("accumulate_ragged_pertap", IG(1, 32, 0, 0, 16), H=13, W=11, Cout=96, act=0, fmt="f16", feats={"accumulate", "pmul"}),
    # ---- depth: calibrates sqrt(K)
    case("deep_cin1024_tf32", IG(0, 64, 0, 0, 16), H=4, W=4, Cin=1024, act=0, feats={"bias"}),
    case("deep_cin1024_bf16split", IG(2, 32, 1, 0, 16), H=4, W=4, Cin=1024, Cout=32, act=0, fmt="bf16", split=True),
]


def _variant_case(kernel, fmt, bn, merged, spec, cw, reg):
    """A case that selects the given instantiation: plain conv (two N tiles) for SPEC 0, SPADE with bf16 hi/lo only for SPEC 1/2."""
    f = {0: "tf32", 1: "f16", 2: "bf16"}[fmt]
    knobs = {"MG_GROUP3": 0} if kernel == "ig" else {"MG_EPI_REG": int(reg)}
    kw = dict(fmt=f, split=merged, ctas=5)
    if spec:
        kw.update(spade=(bn // 2, 1), act=2 if spec == 1 else 0, out16=("bf16", True), want_f32=False)
        if cw == 32:
            knobs["MG_EPI_CW_SPADE"] = 32
    else:
        kw.update(Cout=2 * bn, bn=bn, feats={"bias", "res"})
        if cw == 32:
            knobs["MG_EPI_CW16"] = 0
    if kernel == "ig":
        kw.update(H=12, W=20)          # ragged in both tile dimensions, not eligible for the group kernel
        v = IG(fmt, bn, merged, spec, cw)
    else:
        kw.update(H=16, W=32)
        v = G3(fmt, bn, merged, spec, cw, reg)
    return case("variant_" + re.sub(r"[^0-9a-z]+", "_", v.split("_kernel")[0] + v.split("kernel")[1]).strip("_"), v,
                knobs=knobs, **kw)


def _all_variants():
    """Every (kernel, FMT, BN, MERGED, SPEC, CW, REG) the launchers can select (conv_variant_exists, conv3_reg_epilogue)."""
    out = []
    for fmt in (0, 1, 2):
        for bn in (32, 64, 128):
            for merged in (False, True):
                for spec in (0, 1, 2):
                    for cw in (16, 32):
                        ok = (not merged or (fmt != 0 and 2 * bn <= 128)) and (spec == 0 or bn % 64 == 0) and \
                             (cw == 16 or (bn >= 64 if spec == 0 else bn == 128))
                        if not ok:
                            continue
                        out.append(("ig", fmt, bn, merged, spec, cw, False))
                        out.append(("g3", fmt, bn, merged, spec, cw, False))
                        if cw == 16 and not (bn == 128 and not merged and spec == 0):
                            out.append(("g3", fmt, bn, merged, spec, cw, True))
    return out


def _variant_name(v):
    kernel, fmt, bn, merged, spec, cw, reg = v
    return IG(fmt, bn, merged, spec, cw) if kernel == "ig" else G3(fmt, bn, merged, spec, cw, reg)


_covered = {c["variant"] for c in HAND}
CASES = HAND + [_variant_case(*v) for v in _all_variants()
                if _variant_name(v) not in _covered and _variant_name(v) not in UNREACHABLE]


# ============================================================================================== CPU: variant coverage
def test_every_compiled_conv_variant_is_exercised():
    """The library's igemm_tf32_kernel / conv3x3_group_kernel instantiations (nm -C) = the expected variants of the cases
    above plus UNREACHABLE.  A new instantiation needs a case; a case whose variant is not compiled is wrong."""
    from michigan_b200 import _lib as lib_mod
    nm = shutil.which("nm")
    assert nm, "nm (binutils) is needed to list the library's kernels"
    assert os.path.exists(lib_mod.LIB_PATH), "build the library first (python -m michigan_b200.build)"
    r = subprocess.run([nm, "-C", "--defined-only", lib_mod.LIB_PATH], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    found = {_norm(m.group(0)) for line in r.stdout.splitlines() for m in [KERNEL_RE.search(line)] if m}
    assert len(found) > 0
    expected = {c["variant"] for c in CASES}
    assert len({c["name"] for c in CASES}) == len(CASES)
    assert not expected & set(UNREACHABLE), sorted(expected & set(UNREACHABLE))
    assert expected <= found, sorted(expected - found)
    assert set(UNREACHABLE) <= found, sorted(set(UNREACHABLE) - found)
    assert found <= expected | set(UNREACHABLE), sorted(found - expected - set(UNREACHABLE))


# ============================================================================================== GPU: the cases
def _launched(fn):
    """fn() under torch.profiler -> (result, set of conv kernel instantiations launched, names of all CUDA kernels)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    kernels = {ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
    names = {_norm(m.group(0)) for n in kernels for m in [KERNEL_RE.search(n)] if m}
    return res, names, kernels


def _with_knobs(knobs, fn):
    lib, prev = _lib(), {}
    try:
        for k_, v_ in knobs.items():
            prev[k_] = lib.set_tuning(k_, v_)
        return fn()
    finally:
        for k_, v_ in reversed(list(prev.items())):
            lib.set_tuning(k_, v_)


def _make(c):
    """Inputs (CPU fp32), packed weights (device) and the reference weight parts of a case."""
    ops = _ops()
    g = torch.Generator().manual_seed(zlib.crc32(c["name"].encode()))
    rn = lambda *s: torch.randn(*s, generator=g)
    ru = lambda *s: torch.rand(*s, generator=g)
    fmt, split, N, H, W, Cin, k = c["fmt"], c["split"], c["N"], c["H"], c["W"], c["Cin"], c["k"]
    pad_h = c["p"] + (c["extra"] or {}).get("pad_h_extra", 0)
    pad_w = c["p"] + (c["extra"] or {}).get("pad_w_extra", 0)
    if c["out_hw"]:
        OH, OW = c["out_hw"]
    else:
        OH, OW = (H + 2 * c["p"] - k) // c["s"] + 1, (W + 2 * c["p"] - k) // c["s"] + 1
    Cout = c["spade"][0] if c["spade"] else c["Cout"]
    d = dict(OH=OH, OW=OW, Cout=Cout, pad_h=pad_h, pad_w=pad_w)
    x32 = rn(N, H, W, Cin)
    if fmt == "tf32":
        acts = [rna_tf32(x32)]
        d["x"], d["x_lo"] = acts[0].to(dev), None
    elif split:
        acts = list(split16(x32, fmt))
        d["x"], d["x_lo"] = acts[0].to(dev), acts[1].to(dev)
    else:
        acts = [x32.to(T16[fmt])]
        d["x"], d["x_lo"] = acts[0].to(dev), None
    d["acts"], d["x32"] = acts, x32
    wscale = 1.0 / (k * k * Cin) ** 0.5
    if c["spade"]:
        C, xs = c["spade"]
        wg, wb = rn(C, Cin, k, k) * wscale, rn(C, Cin, k, k) * wscale
        bn = ops.spade_bn(C)
        if fmt == "tf32":
            wp = ops.pack_weight_gb(wg.to(dev), wb.to(dev))
        else:
            wp = ops.pack_weight_gb16(wg.to(dev), wb.to(dev), FMT[fmt], split=split)
        exp, d["wg_parts"], d["wb_parts"] = packed_gb(wg, wb, fmt, split, bn)
        d["spade_in"] = (rn(N, OH >> xs, OW >> xs, C), xs, ru(C) + 0.5, rn(C), 1 + 0.2 * rn(C), 0.3 * rn(C))
    else:
        w = rn(Cout, Cin, k, k) * wscale
        if "zero" in c["feats"]:
            w[:8] = 0
        inv = None if c["inv"] is None else torch.tensor([c["inv"]], dtype=torch.float32)
        invd = None if inv is None else inv.to(dev)
        if fmt == "tf32":
            wp = ops.pack_weight(w.to(dev), invd, round_tf32=True)
        else:
            wp = ops.pack_weight16(w.to(dev), invd, FMT[fmt], split=split)
        exp, d["w_parts"] = packed(w, fmt, split, inv)
    _same_bits("%s: packed weights" % c["name"], wp, exp)
    d["wp"] = wp
    f = c["feats"]
    if "bias" in f:
        b = 0.5 * rn(Cout)
        if "zero" in f:
            b[:8] = torch.tensor([0.0, -0.0] * 4)
        if "big" in f:
            # fp16 outputs beyond 65504: hi saturates, lo = cvt(y - 65504) is finite up to |y| = 131008 and +-inf above
            b[:12] = torch.tensor([7e4, -7e4, 1.2e5, -1.2e5, 1.31e5, -1.31e5, 1.32e5, -1.32e5, 3e5, -3e5, 6.5e4, -6.55e4])
        d["bias"] = b
    if "res" in f:
        d["res"], d["rs"] = rn(N, OH, OW, Cout), 0
    if "res1" in f:
        d["res"], d["rs"] = rn(N, OH >> 1, OW >> 1, Cout), 1
    if "pscale" in f:
        d["pscale"] = ru(N, OH, OW) + 0.5
    if "pmul" in f:
        pm = ru(N, OH, OW)
        pm[pm < 0.2] = 0.0
        d["pmul"] = pm
    for ms in (1, 2, 4):
        if ("blend%d" % ms if ms > 1 else "blend") in f:
            hair, back = ru(N, OH * ms, OW * ms), ru(N, OH * ms, OW * ms)
            hair[:, ::3] = 1.0
            back[:, 1::4] = 0.0
            d["blend"] = (rn(N, OH, OW, Cout), hair, back, ms)
    return d


def _run(c, d, round_out=None, want_f32=None, out16="case"):
    """One conv_igemm call of case c -> dict of CPU result tensors (out, hi, lo, aux)."""
    ops = _ops()
    f = c["feats"]
    OH, OW, Cout = d["OH"], d["OW"], d["Cout"]
    cu = lambda t: None if t is None else t.to(dev)
    want_f32 = c["want_f32"] if want_f32 is None else want_f32
    o16 = c["out16"] if out16 == "case" else out16
    kw = dict(act=c["act"], round_out=c["round"] if round_out is None else round_out, bn=c["bn"], max_ctas=c["ctas"],
              a_fmt=FMT[c["fmt"]], x_lo=d["x_lo"], want_f32=want_f32, out16=None if o16 is None else (FMT[o16[0]], o16[1]))
    kw["bias"], kw["pscale"], kw["pmul"] = cu(d.get("bias")), cu(d.get("pscale")), cu(d.get("pmul"))
    if "res" in d:
        kw["res"], kw["res_shift"] = cu(d["res"]), d["rs"]
    if "blend" in d:
        bf, hair, back, ms = d["blend"]
        kw["blend"] = (cu(bf), cu(hair), cu(back), ms)
    if c["spade"]:
        xs_t, xs, sc, sh, g1, bb = d["spade_in"]
        kw["spade"] = (cu(xs_t), xs, cu(sc), cu(sh), cu(g1), cu(bb))
        if "aux" in f:
            kw["aux"] = torch.full((c["N"], OH, OW, Cout), float("nan"), device=dev)
    if c["extra"]:
        kw["_extra"] = dict(c["extra"], accumulate=int("accumulate" in f))
        kw["out_hw"] = (OH, OW)
        shape = (c["N"], c["extra"]["OHF"], c["extra"]["OWF"], Cout)
    else:
        kw["_extra"] = {"accumulate": int("accumulate" in f)}
        shape = (c["N"], OH, OW, Cout)
    if want_f32:
        kw["out"] = d["out0"].to(dev) if "out0" in d else torch.full(shape, float("nan"), device=dev)
    r = ops.conv_igemm(d["x"], d["wp"], Cout, c["k"], c["k"], c["s"], c["p"], **kw)
    out, hi, lo = r if isinstance(r, tuple) else (r, None, None)
    torch.cuda.synchronize()
    res = dict(out=out, hi=hi, lo=lo, aux=kw.get("aux"))
    return {k_: v_.cpu() for k_, v_ in res.items() if v_ is not None}


def _reference(c, d):
    """fp64 reference of the case's fp32 output (ref, R_abs, K), and of the SPADE 1 + gamma copy."""
    OH, OW, s = d["OH"], d["OW"], c["s"]
    nparts = 3 if c["split"] else 1
    K = c["k"] * c["k"] * c["Cin"] * nparts
    acts = d["acts"]

    def pairs(wparts):
        if c["split"]:
            return [(acts[0], wparts[0]), (acts[1], wparts[0]), (acts[0], wparts[1])]
        return [(acts[0], wparts[0])]

    gemm = lambda wp: gemm_ref(pairs(wp), s, d["pad_h"], d["pad_w"], OH, OW)
    aux = None
    if c["spade"]:
        xs_t, xs, sc, sh, g1, bb = (d64(t) if torch.is_tensor(t) else t for t in d["spade_in"])
        gam, rg = gemm(d["wg_parts"])
        bet, rb = gemm(d["wb_parts"])
        xu = up(xs_t, xs, OH, OW)
        m = xu * sc + sh
        ref = act64(m * (g1 + gam) + (bb + bet), c["act"])
        rabs = ((xu * sc).abs() + sh.abs()) * (g1.abs() + rg) + bb.abs() + rb
        aux = (g1 + gam, g1.abs() + rg)
    else:
        ref, rabs = gemm(d["w_parts"])
        if c["split"]:
            full, _ = gemm_ref([(d["x32"], d["w_parts"][0].float() + d["w_parts"][1].float())], s, d["pad_h"], d["pad_w"], OH, OW)
            print("%s: split precision vs the unsplit operands (dropped A_lo W_lo and operand rounding), max / (u R_g) = %.3g"
                  % (c["name"], float(((ref - full).abs() / (U * rabs + TINY)).max())))
        if "pscale" in d:
            ps = d64(d["pscale"])[..., None]
            ref, rabs = ref * ps, rabs * ps.abs()
        if "bias" in d:
            b = d64(d["bias"])
            ref, rabs = ref + b, rabs + b.abs()
        if "res" in d:
            r = up(d64(d["res"]), d["rs"], OH, OW)
            ref, rabs = ref + r, rabs + r.abs()
        ref = act64(ref, c["act"])
        if "blend" in d:
            bf, hair, back, ms = d["blend"]
            om_h = 1 - d64(hair)[:, ::ms, ::ms][:, :OH, :OW, None]
            om_b = 1 - d64(back)[:, ::ms, ::ms][:, :OH, :OW, None]
            ref = om_h * d64(bf) + om_b * ref
            rabs = om_b.abs() * rabs + om_h.abs() * d64(bf).abs()
        if "pmul" in d:
            pm = d64(d["pmul"])[..., None]
            ref, rabs = ref * pm, rabs * pm.abs()
    return ref, rabs, K, aux


def _window(c, d, ref, rabs):
    """Place the (OH, OW) result into the output tensor the kernel writes: strided window, accumulation onto out0."""
    acc = "accumulate" in c["feats"]
    if not c["extra"] and not acc:
        return ref, rabs, None
    out0 = d64(d["out0"])
    if not c["extra"]:
        return out0 + ref, out0.abs() + rabs, None
    e = c["extra"]
    os_, OH, OW = e["out_stride"], d["OH"], d["OW"]
    hs = slice(e["out_off_h"], e["out_off_h"] + os_ * (OH - 1) + 1, os_)
    ws = slice(e["out_off_w"], e["out_off_w"] + os_ * (OW - 1) + 1, os_)
    full, fr = out0.clone(), torch.zeros_like(out0)
    owned = torch.zeros(out0.shape[:3], dtype=torch.bool)
    owned[:, hs, ws] = True
    full[:, hs, ws] = (out0[:, hs, ws] if acc else 0) + ref
    fr[:, hs, ws] = (out0[:, hs, ws].abs() if acc else 0) + rabs
    return full, fr, owned


def _check_16(name, hi, lo, ref, rabs, fmt, k):
    """16-bit-only output against the reference: hi (+ lo) within the format's rounding of the fp32 value plus k u R_abs."""
    bits = 11 if fmt == "f16" else 8
    v = d64(hi) + (d64(lo) if lo is not None else 0)
    rel = 2.0 ** -(2 * bits if lo is not None else bits)
    tiny16 = 2.0 ** -25 if fmt == "f16" else 0.0          # fp16 subnormal spacing / 2
    assert bool(torch.isfinite(v).all()), name
    err = (v - ref).abs()
    bound = k * U * rabs + rel * (ref.abs() + k * U * rabs) + tiny16 * (2 if lo is not None else 1) + TINY
    ratio = float(((err - rel * ref.abs()).clamp_min(0) / (U * rabs + TINY)).max())
    print("%s: max (|hi+lo - ref| - format rounding) / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > bound
    assert not bool(bad.any()), (name, int(bad.sum()), tuple(bad.nonzero()[0].tolist()))


@pytest.mark.gpu
@pytest.mark.parametrize("c", [pytest.param(c, id=c["name"]) for c in CASES])
def test_conv_forward_fp64(c):
    c = dict(c, round="round" in c["feats"])
    assert not (c["round"] and "accumulate" in c["feats"])
    d = _make(c)
    if "accumulate" in c["feats"] or c["extra"]:
        e = c["extra"]
        shape = (c["N"], e["OHF"], e["OWF"], d["Cout"]) if e else (c["N"], d["OH"], d["OW"], d["Cout"])
        d["out0"] = torch.randn(*shape, generator=torch.Generator().manual_seed(5))
    name = c["name"]

    # CUPTI now and then delivers no record of the conv kernel for a short profiling session: profile again then (a reroute
    # to another variant still fails: it shows up under its own name)
    for _ in range(3):
        r1, launched, kernels = _with_knobs(c["knobs"], lambda: _launched(lambda: _run(c, d)))
        if launched:
            break
    assert launched == {c["variant"]}, (name, c["variant"], launched, sorted(kernels))
    r2 = _with_knobs(c["knobs"], lambda: _run(c, d))
    for key in r1:
        _same_bits("%s: %s, second run" % (name, key), r1[key], r2[key])

    ref, rabs, K, aux = _reference(c, d)
    k = C_GEMM * K ** 0.5 + K_EPI
    ref_o, rabs_o, owned = _window(c, d, ref, rabs)
    ratio = 0.0
    if "out" in r1:
        out = r1["out"]
        if owned is not None:
            _same_bits("%s: elements outside the output window" % name, out[~owned], d["out0"][~owned])
        if c["round"]:
            assert not bool((out.view(torch.int32) & 0x1FFF).any()), name
            plain = _with_knobs(c["knobs"], lambda: _run(c, d, round_out=False))
            _same_bits("%s: round_out = rna_tf32 of the unrounded output" % name, out, rna_tf32(plain["out"]))
            ratio = check_rounded(name, out, ref_o, rabs_o, 11, k)
        else:
            ratio = check_close(name, out, ref_o, rabs_o, k)
        if "hi" in r1:
            fmt16 = c["out16"][0]
            hi, lo = split16(out, fmt16)
            _same_bits("%s: hi = cvt(y32)" % name, r1["hi"], hi)
            if "lo" in r1:
                _same_bits("%s: lo = cvt(y32 - hi)" % name, r1["lo"], lo)
            if fmt16 == "f16":
                big = out.abs() > 65504
                assert bool((r1["hi"][big].float().abs() == 65504).all()), name
                if "lo" in r1:
                    # the documented contract: lo overflows to +-inf exactly where y - float(hi) is beyond fp16's range
                    assert torch.equal(torch.isinf(r1["lo"]), (out - r1["hi"].float()).abs() >= 65520), name
                    if "big" in c["feats"]:
                        assert bool(torch.isinf(r1["lo"]).any()) and bool(big.any()), name
    else:
        fmt16 = c["out16"][0]
        _check_16(name, r1["hi"], r1.get("lo"), ref_o, rabs_o, fmt16, k)
        if c["spade"]:
            # SPEC 1 / 2 against the generic variant on the same operands (same MMAs, fp32 output + 16-bit copies)
            gen = _with_knobs(c["knobs"], lambda: _run(c, d, want_f32=True))
            hi, lo = split16(gen["out"], fmt16)
            _same_bits("%s: hi = split of the generic variant's output" % name, r1["hi"], hi)
            _same_bits("%s: lo = split of the generic variant's output" % name, r1["lo"], lo)
            _same_bits("%s: hi, generic variant" % name, gen["hi"], hi)
    if "aux" in r1:
        check_close(name + ": aux (1 + gamma)", r1["aux"], aux[0], aux[1], k)
    print("CASE %-40s %-48s K=%-6d max ratio %.3g  / sqrt(K) %.3g  k %.1f" % (name, c["variant"], K, ratio, ratio / K ** 0.5, k))


# ============================================================================================== refusals
@pytest.mark.gpu
def test_refusals_return_errors():
    """Arguments the ABI refuses return an error status and leave the output untouched."""
    ops, lib = _ops(), _lib()
    g = torch.Generator().manual_seed(3)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev)
    # SPADE C = 96: 2C = 192 is not a multiple of spade_bn(96) = 128, so the [gamma | beta] tiles cannot be packed
    wg, wb = rn(96, 64, 3, 3), rn(96, 64, 3, 3)
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        ops.pack_weight_gb(wg, wb)
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        ops.pack_weight_gb16(wg, wb, ops.F16)
    # a strided output window supports the plain bias epilogue only
    x = rna_tf32(rn(2, 8, 8, 32).cpu()).to(dev)
    wp = ops.pack_weight(rn(64, 32, 3, 3))
    out = torch.full((2, 16, 16, 64), float("nan"), device=dev)
    with pytest.raises(lib.MichiganNativeError, match=r"status -8"):
        ops.conv_igemm(x, wp, 64, 3, 3, 1, 1, out=out, out_hw=(8, 8), res=rn(2, 8, 8, 64),
                       _extra=dict(out_stride=2, OHF=16, OWF=16))
    assert bool(out.isnan().all())
    # Cin not a multiple of the K chunk: 32 for TF32, 64 for 16-bit operands
    out = torch.full((2, 8, 8, 64), float("nan"), device=dev)
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        ops.conv_igemm(rn(2, 8, 8, 48), ops.pack_weight(rn(64, 48, 3, 3)), 64, 3, 3, 1, 1, out=out)
    x16 = rn(2, 8, 8, 96).to(torch.bfloat16)
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        ops.conv_igemm(x16, ops.pack_weight16(rn(64, 96, 3, 3), None, ops.BF16, split=False), 64, 3, 3, 1, 1, a_fmt=ops.BF16, out=out)
    torch.cuda.synchronize()
    assert bool(out.isnan().all())
