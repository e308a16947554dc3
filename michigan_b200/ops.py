"""Functional wrappers: torch CUDA tensors in, C-ABI calls on the current stream, torch tensors out.

PyTorch is plumbing here (device memory, streams); every arithmetic op below runs in
libmichigan_sm90.so.  Activations are NHWC fp32 ([N,H,W,C] contiguous).
"""
import ctypes as C
import math

import torch

from . import _lib
from ._lib import IgemmArgs, ThinArgs, check

ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH = 0, 1, 2, 3
EPI_BIAS, EPI_SPADE = 0, 1
# tensor-core operand formats
TF32, F16, BF16 = 0, 1, 2
_T16 = {F16: torch.float16, BF16: torch.bfloat16}


def _dt(fmt):
    return torch.float32 if fmt == TF32 else _T16[fmt]


def _alloc16(shape, device, out16):
    """out16 = None | (fmt, want_lo) -> (hi, lo) tensors (or None)."""
    if out16 is None:
        return None, None
    fmt, want_lo = out16
    hi = torch.empty(shape, device=device, dtype=_T16[fmt])
    lo = torch.empty(shape, device=device, dtype=_T16[fmt]) if want_lo else None
    return hi, lo


def _p(t):
    if t is None:
        return None
    return t.data_ptr()


def _stream():
    """Raw cudaStream_t of torch's current stream (the C accessor: ~0.3 us instead of ~14 us for the Stream object)."""
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def _chk(t, name, dtype=torch.float32):
    if t is None:
        return
    if not t.is_cuda:
        raise _lib.MichiganNativeError("%s must be a CUDA tensor (no CPU path exists)" % name)
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)


# widest GEMM N tile of the implicit-GEMM kernels (128 accumulator columns per consumer warpgroup)
_SPADE_BN_MAX = 128


def spade_bn(c):
    """GEMM N tile used for a gamma|beta operand of `c` channels (must match the weight packing: [gamma(BN/2) | beta(BN/2)] per
    N tile)."""
    return _SPADE_BN_MAX if 2 * c >= _SPADE_BN_MAX else max(64, 2 * c)


# ------------------------------------------------------------------------------------------ weights
def pack_weight(w_oihw, inv_sigma=None, round_tf32=True):
    _chk(w_oihw, "w"); _chk(inv_sigma, "inv_sigma")
    O, I, KH, KW = w_oihw.shape
    out = torch.empty((O, KH * KW * I), device=w_oihw.device, dtype=torch.float32)
    check(_lib.load().mg_pack_weight(_p(w_oihw), _p(out), O, I, KH, KW, _p(inv_sigma), int(round_tf32), _stream()),
          "mg_pack_weight")
    return out


def pack_weight_gb(wg, wb):
    _chk(wg, "wg"); _chk(wb, "wb")
    Cc, I, KH, KW = wg.shape
    bn = spade_bn(Cc)
    out = torch.empty((2 * Cc, KH * KW * I), device=wg.device, dtype=torch.float32)
    check(_lib.load().mg_pack_weight_gb(_p(wg), _p(wb), _p(out), Cc, I, KH, KW, bn, _stream()), "mg_pack_weight_gb")
    return out


def pack_weight16(w_oihw, inv_sigma=None, fmt=BF16, split=True):
    """16-bit operand [O][tap][hi|lo][I] (lo only when split) of w * inv_sigma."""
    _chk(w_oihw, "w"); _chk(inv_sigma, "inv_sigma")
    O, I, KH, KW = w_oihw.shape
    out = torch.empty((O, KH * KW * (2 if split else 1) * I), device=w_oihw.device, dtype=_T16[fmt])
    check(_lib.load().mg_pack_weight16(_p(w_oihw), _p(out), O, I, KH, KW, _p(inv_sigma), fmt, int(split), _stream()),
          "mg_pack_weight16")
    return out


def pack_weight_gb16(wg, wb, fmt=F16, split=False):
    _chk(wg, "wg"); _chk(wb, "wb")
    Cc, I, KH, KW = wg.shape
    out = torch.empty((2 * Cc, KH * KW * I * (2 if split else 1)), device=wg.device, dtype=_T16[fmt])
    check(_lib.load().mg_pack_weight_gb16(_p(wg), _p(wb), _p(out), Cc, I, KH, KW, spade_bn(Cc), fmt, int(split), _stream()),
          "mg_pack_weight_gb16")
    return out


def pack_weight_thin(w_oihw, cin_pad):
    _chk(w_oihw, "w")
    O, I, KH, KW = w_oihw.shape
    out = torch.empty((KH * KW, cin_pad, O), device=w_oihw.device, dtype=torch.float32)
    check(_lib.load().mg_pack_weight_thin(_p(w_oihw), _p(out), O, I, cin_pad, KH, KW, _stream()), "mg_pack_weight_thin")
    return out


# ------------------------------------------------------------------------------------------ convs
def conv_igemm(x, wpack, cout, kh, kw, stride=1, pad=0, *, act=ACT_NONE, round_out=False, bias=None, res=None,
               res_shift=0, pscale=None, pmul=None, blend=None, spade=None, bn=0, max_ctas=0, out=None, out_hw=None, _extra=None,
               a_fmt=TF32, x_lo=None, out16=None, want_f32=True, aux=None):
    """Implicit-GEMM conv on wgmma.  x: [N,H,W,Cin]; returns [N,OH,OW,cout].

    blend = (bf[N,OH,OW,cout], hair[N,MH,MW], back[N,MH,MW], mask_stride)
    spade = (xsrc[N,OH>>s,OW>>s,cout], x_shift, nscale[c], nshift[c], gbias1[c], bbias[c])
    a_fmt: operand format of x / wpack (TF32 = fp32 storage, F16, BF16); x_lo: low part -> 3-pass split
    precision (wpack from pack_weight16(split=True)).  out16=(fmt, want_lo): also emit 16-bit copies of
    the result; with want_f32=False only those.  Returns out32, or (out32|None, hi, lo|None) with out16.
    """
    _chk(x, "x", _dt(a_fmt)); _chk(wpack, "wpack", _dt(a_fmt)); _chk(x_lo, "x_lo", _dt(a_fmt)); _chk(bias, "bias"); _chk(res, "res"); _chk(pscale, "pscale"); _chk(pmul, "pmul")
    N, H, W, Cin = x.shape
    if out_hw is not None:
        OH, OW = out_hw
    else:
        OH = (H + 2 * pad - kh) // stride + 1
        OW = (W + 2 * pad - kw) // stride + 1
    if out is None and want_f32:
        out = torch.empty((N, OH, OW, cout), device=x.device, dtype=torch.float32)
    hi, lo = _alloc16((N, OH, OW, cout), x.device, out16)
    a = IgemmArgs()
    a.inp, a.wpack, a.out = _p(x), _p(wpack), _p(out)
    a.a_fmt, a.split, a.in_lo = a_fmt, int(x_lo is not None), _p(x_lo)
    a.out_hi, a.out_lo, a.out16_fmt = _p(hi), _p(lo), (out16[0] if out16 else 0)
    a.aux_out = _p(aux)
    a.N, a.H, a.W, a.Cin = N, H, W, Cin
    a.OH, a.OW, a.Cout = OH, OW, cout
    a.KH, a.KW, a.stride, a.pad = kh, kw, stride, pad
    a.BN = bn
    a.epi = EPI_SPADE if spade is not None else EPI_BIAS
    a.act, a.round_out = act, int(round_out)
    a.bias, a.res, a.res_shift = _p(bias), _p(res), res_shift
    a.pscale, a.pmul = _p(pscale), _p(pmul)
    if res is not None:
        assert tuple(res.shape) == (N, OH >> res_shift, OW >> res_shift, cout), (res.shape, (N, OH, OW, cout), res_shift)
    if blend is not None:
        bf, hair, back, ms = blend
        _chk(bf, "bf"); _chk(hair, "hair"); _chk(back, "back")
        assert tuple(bf.shape) == (N, OH, OW, cout), (bf.shape, (N, OH, OW, cout))
        a.bf, a.hair, a.back = _p(bf), _p(hair), _p(back)
        a.mask_stride, a.MH, a.MW = ms, hair.shape[-2], hair.shape[-1]
    if spade is not None:
        xs, x_shift, nscale, nshift, gbias1, bbias = spade
        for t, nm in ((xs, "spade.x"), (nscale, "nscale"), (nshift, "nshift"), (gbias1, "gbias1"), (bbias, "bbias")):
            _chk(t, nm)
        assert tuple(xs.shape) == (N, OH >> x_shift, OW >> x_shift, cout), (xs.shape, (N, OH, OW, cout), x_shift)
        assert wpack.shape[0] == 2 * cout
        a.x, a.x_shift = _p(xs), x_shift
        a.nscale, a.nshift, a.gbias1, a.bbias = _p(nscale), _p(nshift), _p(gbias1), _p(bbias)
        if bn == 0:
            a.BN = spade_bn(cout)
    else:
        assert wpack.shape[0] == cout, (wpack.shape, cout)
    assert wpack.shape[1] == kh * kw * Cin * (2 if x_lo is not None else 1), (wpack.shape, kh, kw, Cin)
    a.max_ctas = max_ctas
    if _extra is not None:
        for k_, v_ in _extra.items():
            setattr(a, k_, v_)
    check(_lib.load().mg_conv_igemm(C.byref(a), _stream()), "mg_conv_igemm")
    if out16 is not None:
        return out, hi, lo
    return out


def conv_thin(x, wt, bias, cout, kh, kw, stride=1, pad=0, *, pad_mode=0, seg_resize=0, act=ACT_NONE, round_out=False,
              pscale=None, pmul=None, out_hw=None, out16=None, want_f32=True):
    """Direct conv for 3/4/7-channel inputs (channels padded to 4 or 8).  x: [N,H,W,CinP].
    out16=(fmt, want_lo): also write 16-bit copies; returns (out32|None, hi, lo|None) then."""
    _chk(x, "x"); _chk(wt, "wt"); _chk(bias, "bias"); _chk(pscale, "pscale"); _chk(pmul, "pmul")
    N, Hp, Wp, CinP = x.shape
    if seg_resize:
        H, W = out_hw  # virtual (resized) input == output size for the 3x3/pad1 SPADE conv
    else:
        H, W = Hp, Wp
    OH = (H + 2 * pad - kh) // stride + 1
    OW = (W + 2 * pad - kw) // stride + 1
    out = torch.empty((N, OH, OW, cout), device=x.device, dtype=torch.float32) if want_f32 else None
    hi, lo = _alloc16((N, OH, OW, cout), x.device, out16)
    a = ThinArgs()
    a.inp, a.w, a.bias, a.out = _p(x), _p(wt), _p(bias), _p(out)
    a.out_hi, a.out_lo, a.out16_fmt = _p(hi), _p(lo), (out16[0] if out16 else 0)
    a.N, a.H, a.W, a.CinP = N, H, W, CinP
    a.OH, a.OW, a.Cout = OH, OW, cout
    a.KH, a.KW, a.stride, a.pad = kh, kw, stride, pad
    a.pad_mode, a.seg_resize = pad_mode, seg_resize
    a.act, a.round_out = act, int(round_out)
    a.pscale, a.pmul = _p(pscale), _p(pmul)
    check(_lib.load().mg_conv_thin(C.byref(a), _stream()), "mg_conv_thin")
    if out16 is not None:
        return out, hi, lo
    return out


def dog_response(img_nchw, bank, hair):
    """The DoG orientation response pass of L1OLoss (mg_conv_thin's arg-max epilogue): img [N,3,H,W] in [-1,1], bank the
    [17*17][32] filters, hair [N,H,W] -> (idx [N,H,W] uint8 first arg-max of the clamped responses, rh [N,H,W] = max response *
    hair, m [1] = max of rh over the batch, on the device)."""
    _chk(img_nchw, "img"); _chk(bank, "bank"); _chk(hair, "hair")
    N, _, H, W = img_nchw.shape
    idx = torch.empty((N, H, W), device=img_nchw.device, dtype=torch.uint8)
    rh = torch.empty((N, H, W), device=img_nchw.device, dtype=torch.float32)
    m = torch.zeros(1, device=img_nchw.device, dtype=torch.float32)
    a = ThinArgs()
    a.inp, a.w, a.out = _p(img_nchw), _p(bank), _p(rh)
    a.N, a.H, a.W, a.CinP = N, H, W, 3
    a.OH, a.OW, a.Cout = H, W, 32
    a.KH, a.KW, a.stride, a.pad = 17, 17, 1, 8
    a.argmax_idx, a.argmax_mask, a.argmax_max = _p(idx), _p(hair), _p(m)
    check(_lib.load().mg_conv_thin(C.byref(a), _stream()), "mg_conv_thin")
    return idx, rh, m


def pack_weight_seg_tc(w_oihw):
    """bf16 [128][128] operand of conv_seg_tc: k = part*36 + tap*4 + ci with parts (W_hi, W_hi, W_lo)."""
    _chk(w_oihw, "w")
    O, I, KH, KW = w_oihw.shape
    assert KH == 3 and KW == 3
    out = torch.empty((O, 128), device=w_oihw.device, dtype=torch.bfloat16)
    check(_lib.load().mg_pack_weight_seg_tc(_p(w_oihw), _p(out), O, I, _stream()), "mg_pack_weight_seg_tc")
    return out


def conv_seg_tc(seg4, wpack, bias, *, seg_resize=0, act=ACT_RELU, round_out=False, out_hw=None, out16=None, want_f32=True):
    """SPADE mlp_shared (4 -> 128, 3x3, pad 1, + act) on tensor cores; same results contract as conv_thin."""
    _chk(seg4, "seg4"); _chk(wpack, "wpack", torch.bfloat16); _chk(bias, "bias")
    N, Hp, Wp, CinP = seg4.shape
    H, W = out_hw if seg_resize else (Hp, Wp)
    out = torch.empty((N, H, W, 128), device=seg4.device, dtype=torch.float32) if want_f32 else None
    hi, lo = _alloc16((N, H, W, 128), seg4.device, out16)
    a = ThinArgs()
    a.inp, a.w, a.bias, a.out = _p(seg4), _p(wpack), _p(bias), _p(out)
    a.out_hi, a.out_lo, a.out16_fmt = _p(hi), _p(lo), (out16[0] if out16 else 0)
    a.N, a.H, a.W, a.CinP = N, H, W, CinP
    a.OH, a.OW, a.Cout = H, W, 128
    a.KH, a.KW, a.stride, a.pad = 3, 3, 1, 1
    a.pad_mode, a.seg_resize = 0, seg_resize
    a.act, a.round_out = act, int(round_out)
    check(_lib.load().mg_conv_seg_tc(C.byref(a), _stream()), "mg_conv_seg_tc")
    if out16 is not None:
        return out, hi, lo
    return out


def pack_mlp_shared(w_oihw):
    """Operand of SPADE's mlp_shared conv (label_nc <= 4 -> 128, 3x3): tensor-core bf16 split, or the thin-conv layout."""
    if w_oihw.shape[0] == 128 and w_oihw.shape[1] <= 4:
        return pack_weight_seg_tc(w_oihw)
    return pack_weight_thin(w_oihw, 4)


def mlp_shared(seg4, wpack, bias, *, seg_resize, out_hw, act=ACT_RELU, round_out=False, out16=None, want_f32=True):
    """actv = act(conv3x3(nearest_resize(seg4)) + b) (normalization.py:110-111), dispatching on the packed operand."""
    if wpack.dtype == torch.bfloat16:
        return conv_seg_tc(seg4, wpack, bias, seg_resize=seg_resize, act=act, round_out=round_out, out_hw=out_hw, out16=out16,
                           want_f32=want_f32)
    return conv_thin(seg4, wpack, bias, 128, 3, 3, 1, 1, seg_resize=seg_resize, act=act, round_out=round_out, out_hw=out_hw,
                     out16=out16, want_f32=want_f32)


def conv_img(x, w_oihw, bias, act_in=ACT_LRELU, act_out=ACT_TANH):
    _chk(x, "x"); _chk(w_oihw, "w"); _chk(bias, "bias")
    N, H, W, Cin = x.shape
    cout = w_oihw.shape[0]
    out = torch.empty((N, cout, H, W), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_conv_img(_p(x), _p(w_oihw), _p(bias), _p(out), N, H, W, Cin, cout, act_in, act_out, _stream()),
          "mg_conv_img")
    return out


def conv_to1(x, w_oihw, bias, pad):
    _chk(x, "x"); _chk(w_oihw, "w"); _chk(bias, "bias")
    N, H, W, Cin = x.shape
    _, _, KH, KW = w_oihw.shape
    OH, OW = H + 2 * pad - KH + 1, W + 2 * pad - KW + 1
    out = torch.empty((N, OH, OW, 1), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_conv_to1(_p(x), _p(w_oihw), _p(bias), _p(out), N, H, W, Cin, KH, KW, pad, _stream()), "mg_conv_to1")
    return out


# ------------------------------------------------------------------------------------------ norms
def bn_sums(x):
    """Per-channel (sum, sum of squares) of an NHWC tensor as a [2*C + 1] float64 tensor; the spare last element carries
    the sample count through the cross-rank exchange (sync_batchnorm.allreduce_sums)."""
    _chk(x, "x")
    Cc = x.shape[-1]
    sums = torch.zeros(2 * Cc + 1, device=x.device, dtype=torch.float64)
    check(_lib.load().mg_bn_stats(_p(x), x.numel() // Cc, Cc, _p(sums), _stream()), "mg_bn_stats")
    return sums


def chan_sum_cvt16(x):
    """-> (per-channel sums [C] fp32, bf16 copy of x) in ONE pass over x (bias gradient + gradient-GEMM operand)."""
    _chk(x, "x")
    Cc = x.shape[-1]
    sums = torch.zeros(2 * Cc + 1, device=x.device, dtype=torch.float64)
    out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    check(_lib.load().mg_bn_stats_cvt16(_p(x), x.numel() // Cc, Cc, _p(sums), _p(out), _stream()), "mg_bn_stats_cvt16")
    return sums[:Cc].float(), out


def bn_finalize(sums, count, unbiased_mult=1, eps=1e-5, momentum=0.1, clamp_mode=0, running_mean=None, running_var=None,
                want_stats=False):
    """count: number of samples behind `sums`, or 0.0 = read the all-reduced count from sums[2*C] on the device;
    unbiased_mult: 4^s when the normalised tensor is the 2^s-upsampled view (running_var's unbiased factor)."""
    Cc = sums.numel() // 2
    nscale = torch.empty(Cc, device=sums.device, dtype=torch.float32)
    nshift = torch.empty(Cc, device=sums.device, dtype=torch.float32)
    mean = torch.empty(Cc, device=sums.device, dtype=torch.float32) if want_stats else None
    var = torch.empty(Cc, device=sums.device, dtype=torch.float32) if want_stats else None
    _chk(running_mean, "running_mean"); _chk(running_var, "running_var")
    if count <= 0 and sums.numel() != 2 * Cc + 1:
        raise ValueError("bn_finalize: a device-side count needs the [2*C + 1] sums layout")
    check(_lib.load().mg_bn_finalize(_p(sums), Cc, float(count), float(unbiased_mult), eps, momentum, clamp_mode,
                                     _p(nscale), _p(nshift), _p(running_mean), _p(running_var), _p(mean), _p(var),
                                     _stream()), "mg_bn_finalize")
    if want_stats:
        return nscale, nshift, mean, var
    return nscale, nshift


def bn_from_running(running_mean, running_var, eps=1e-5):
    _chk(running_mean, "running_mean"); _chk(running_var, "running_var")
    Cc = running_mean.numel()
    nscale = torch.empty(Cc, device=running_mean.device, dtype=torch.float32)
    nshift = torch.empty(Cc, device=running_mean.device, dtype=torch.float32)
    check(_lib.load().mg_bn_from_running(_p(running_mean), _p(running_var), Cc, eps, _p(nscale), _p(nshift), _stream()),
          "mg_bn_from_running")
    return nscale, nshift


def instance_norm_act(x, act=ACT_LRELU, eps=1e-5, round_out=False, pmul=None, out16=None, want_f32=True):
    """InstanceNorm2d(affine=False) followed by an activation, NHWC.  out16 as in conv_igemm."""
    _chk(x, "x"); _chk(pmul, "pmul")
    N, H, W, Cc = x.shape
    sums = torch.zeros((N, 2, Cc), device=x.device, dtype=torch.float64)
    lib = _lib.load()
    check(lib.mg_in_stats(_p(x), N, H * W, Cc, _p(sums), _stream()), "mg_in_stats")
    ss = torch.empty((N, 2, Cc), device=x.device, dtype=torch.float32)
    y = torch.empty_like(x) if want_f32 else None
    hi, lo = _alloc16(tuple(x.shape), x.device, out16)
    check(lib.mg_in_apply(_p(x), _p(sums), _p(ss), _p(y), N, H * W, Cc, eps, act, int(round_out), _p(pmul), _p(hi), _p(lo),
                          (out16[0] if out16 else 0), _stream()), "mg_in_apply")
    if out16 is not None:
        return y, hi, lo
    return y


def softmax_rows(x2d, fmt=TF32, split=False):
    """Row softmax of a [rows, cols] fp32 matrix, emitted as a tensor-core operand: -> (fmt, hi_or_fp32, lo|None)."""
    _chk(x2d, "scores")
    rows, cols = x2d.shape
    lib = _lib.load()
    if fmt == TF32:
        out = torch.empty_like(x2d)
        check(lib.mg_softmax_rows(_p(x2d), rows, cols, _p(out), None, None, 0, 1, _stream()), "mg_softmax_rows")
        return (TF32, out, None)
    hi, lo = _alloc16((rows, cols), x2d.device, (fmt, split))
    check(lib.mg_softmax_rows(_p(x2d), rows, cols, None, _p(hi), _p(lo), fmt, 0, _stream()), "mg_softmax_rows")
    return (fmt, hi, lo)


# ------------------------------------------------------------------------------------------ prep / pooling
def prep_seg(tag_nchw, orient_nchw):
    _chk(tag_nchw, "input_tag"); _chk(orient_nchw, "orient")
    N, _, H, W = tag_nchw.shape
    oc = orient_nchw.shape[1]
    seg4 = torch.empty((N, H, W, 4), device=tag_nchw.device, dtype=torch.float32)
    check(_lib.load().mg_prep_seg(_p(tag_nchw), _p(orient_nchw), oc, _p(seg4), N, H, W, _stream()), "mg_prep_seg")
    return seg4


def prep_dinput(seg4, img_nchw):
    _chk(seg4, "seg4"); _chk(img_nchw, "image")
    N, H, W, _ = seg4.shape
    out = torch.empty((N, H, W, 8), device=seg4.device, dtype=torch.float32)
    check(_lib.load().mg_prep_dinput(_p(seg4), _p(img_nchw), _p(out), N, H, W, _stream()), "mg_prep_dinput")
    return out


def prep_bginput(img_nchw, noise_nchw, back):
    _chk(img_nchw, "image"); _chk(noise_nchw, "noise"); _chk(back, "back_mask")
    N, _, H, W = img_nchw.shape
    out = torch.empty((N, H, W, 4), device=img_nchw.device, dtype=torch.float32)
    check(_lib.load().mg_prep_bginput(_p(img_nchw), _p(noise_nchw), _p(back), _p(out), N, H, W, _stream()),
          "mg_prep_bginput")
    return out


def nchw_to_nhwc(x, cpad=None, pmul=None):
    _chk(x, "x"); _chk(pmul, "pmul")
    N, Cc, H, W = x.shape
    cp = cpad or Cc
    out = torch.empty((N, H, W, cp), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_nchw_to_nhwc(_p(x), _p(out), N, Cc, H, W, cp, _p(pmul), _stream()), "mg_nchw_to_nhwc")
    return out


def partial_mask(mask, k, stride, pad):
    """PartialConv2d mask update: mask [N,H,W] -> (mask_ratio, update_mask) [N,OH,OW]."""
    _chk(mask, "mask")
    N, H, W = mask.shape
    OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    ratio = torch.empty((N, OH, OW), device=mask.device, dtype=torch.float32)
    upd = torch.empty_like(ratio)
    check(_lib.load().mg_partial_mask(_p(mask), _p(ratio), _p(upd), N, H, W, k, stride, pad, _stream()), "mg_partial_mask")
    return ratio, upd


def _mask_hw(mref, mtag, h, w):
    """(MH, MW) of the full-resolution masks of masked_mean_bcast[_bwd]; both must match.  No mask: the map's own size."""
    hw = [tuple(m.shape[-2:]) for m in (mref, mtag) if m is not None]
    if len(set(hw)) > 1:
        raise ValueError("masked_mean_bcast: mref and mtag differ in size: %s" % (hw,))
    return hw[0] if hw else (h, w)


def masked_mean_bcast(x, mref, mtag):
    """out[n,p,c] = mtag[n,p] * sum_q x[n,q,c] mref[n,q] / max(sum_q mref[n,q], 1) on NHWC x, masks [N,MH,MW] read at stride
    MH/h.  mref None: the plain spatial mean; mtag None: broadcast with weight 1."""
    _chk(x, "x"); _chk(mref, "mref"); _chk(mtag, "mtag")
    N, h, w, Cc = x.shape
    MH, MW = _mask_hw(mref, mtag, h, w)
    out = torch.empty_like(x)
    check(_lib.load().mg_masked_mean_bcast(_p(x), _p(mref), _p(mtag), _p(out), N, h, w, Cc, MH, MW, _stream()),
          "mg_masked_mean_bcast")
    return out


def resize_bilinear(x, oh, ow):
    _chk(x, "x")
    N, H, W, Cc = x.shape
    out = torch.empty((N, oh, ow, Cc), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_resize_bilinear(_p(x), _p(out), N, H, W, Cc, oh, ow, _stream()), "mg_resize_bilinear")
    return out


def reflect_pad(x, pad, round_tf32=False, out16=None, want_f32=True):
    _chk(x, "x")
    N, H, W, Cc = x.shape
    shape = (N, H + 2 * pad, W + 2 * pad, Cc)
    out = torch.empty(shape, device=x.device, dtype=torch.float32) if want_f32 else None
    hi, lo = _alloc16(shape, x.device, out16)
    check(_lib.load().mg_reflect_pad(_p(x), _p(out), N, H, W, Cc, pad, int(round_tf32), _p(hi), _p(lo),
                                     (out16[0] if out16 else 0), _stream()), "mg_reflect_pad")
    if out16 is not None:
        return out, hi, lo
    return out


def nhwc_to_nchw(x, c=None):
    _chk(x, "x")
    N, H, W, cp = x.shape
    Cc = c or cp
    out = torch.empty((N, Cc, H, W), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_nhwc_to_nchw(_p(x), _p(out), N, Cc, H, W, cp, _stream()), "mg_nhwc_to_nchw")
    return out


def maxpool_mask(m, k, invert=False):
    """max_pool2d(k, stride 1, pad k//2) of a [N,H,W] map; invert -> 1 - pooled."""
    _chk(m, "mask")
    N, H, W = m.shape
    out = torch.empty_like(m)
    tmp = torch.empty_like(m)
    check(_lib.load().mg_maxpool_mask(_p(m), _p(out), _p(tmp), N, H, W, k, int(invert), _stream()), "mg_maxpool_mask")
    return out


def avgpool3s2(x):
    _chk(x, "x")
    N, H, W, Cc = x.shape
    OH, OW = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    out = torch.empty((N, OH, OW, Cc), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_avgpool3s2(_p(x), _p(out), N, H, W, Cc, OH, OW, _stream()), "mg_avgpool3s2")
    return out


def _fmt16(t):
    """16-bit format code of a tensor (F16 / BF16)."""
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError("expected a float16 or bfloat16 tensor, got %s" % t.dtype)


def _split32(a):
    """fp32 tensor -> (a32, None, 0); 16-bit tensor -> (None, a16, fmt)."""
    if a.dtype == torch.float32:
        _chk(a, "a")
        return a, None, 0
    fmt = _fmt16(a)
    _chk(a, "a", a.dtype)
    return None, a, fmt


def maxpool2(x, out16=None, want_f32=True):
    """2x2 / stride 2 max-pool (floor mode) of an NHWC tensor read as fp32 or 16-bit (x's dtype).
    out16 = fmt: also write the 16-bit operand of the next conv; returns out32, or (out32|None, out16)."""
    x32, x16, xfmt = _split32(x)
    N, H, W, Cc = x.shape
    out = torch.empty((N, H // 2, W // 2, Cc), device=x.device, dtype=torch.float32) if want_f32 else None
    o16 = torch.empty((N, H // 2, W // 2, Cc), device=x.device, dtype=_T16[out16]) if out16 is not None else None
    check(_lib.load().mg_maxpool2_nhwc(_p(x32), _p(x16), xfmt, _p(out), _p(o16), out16 or 0, N, H, W, Cc, _stream()),
          "mg_maxpool2_nhwc")
    if out16 is not None:
        return out, o16
    return out


# ------------------------------------------------------------------------------------------ backward
def conv_wgrad(dy, x, kh, kw, stride=1, pad=0):
    """Packed weight gradient [Cout][kh*kw*Cin] of an implicit-GEMM conv (tensor cores, split-K)."""
    _chk(dy, "dy"); _chk(x, "x")
    N, H, W, Cin = x.shape
    _, OH, OW, Cout = dy.shape
    dw = torch.empty((Cout, kh * kw * Cin), device=x.device, dtype=torch.float32)
    check(_lib.load().mg_conv_wgrad(_p(dy), _p(x), _p(dw), N, H, W, Cin, OH, OW, Cout, kh, kw, stride, pad, _stream()),
          "mg_conv_wgrad")
    return dw


def dgrad_geometry(k, stride, pad, r):
    """Sub-kernel of the transposed conv for output parity r: (k0, J, pad') (see mg_pack_weight_dgrad)."""
    k0 = (r + pad) % stride
    J = (k - k0 + stride - 1) // stride
    d0 = (r + pad - k0) // stride
    return k0, J, J - 1 - d0


def conv_dgrad(dy, w_oihw, in_hw, stride=1, pad=0, inv_sigma=None, out=None, accumulate=False, dy16=None):
    """dX [N,H,W,Cin] of y = conv(x, w, stride, pad) given dY [N,OH,OW,Cout]; wgmma implicit GEMM on dY
    with flipped/transposed (sub-)kernels, one launch per output parity class (stride^2).
    dy16: bf16 copy of dY -> the GEMM runs with bf16 operands (weights converted after packing), fp32 accumulation."""
    _chk(dy, "dy"); _chk(w_oihw, "w"); _chk(dy16, "dy16", torch.bfloat16)
    if dy16 is not None and (dy.shape[-1] % 64 != 0):
        dy16 = None
    N, OH, OW, Cout = dy.shape
    O, I, KH, KW = w_oihw.shape
    H, W = in_hw
    if out is None:
        out = torch.empty((N, H, W, I), device=dy.device, dtype=torch.float32)
        if stride > 1 and (H < stride or W < stride):
            out.zero_()
    lib = _lib.load()
    for rh in range(stride):
        k0h, Jh, ph = dgrad_geometry(KH, stride, pad, rh)
        for rw in range(stride):
            k0w, Jw, pw = dgrad_geometry(KW, stride, pad, rw)
            ah, aw = (H - rh + stride - 1) // stride, (W - rw + stride - 1) // stride
            if ah <= 0 or aw <= 0:
                continue
            if Jh <= 0 or Jw <= 0:
                if not accumulate:
                    out[:, rh::stride, rw::stride].zero_()
                continue
            wp = torch.empty((I, Jh * Jw * O), device=dy.device, dtype=torch.float32)
            check(lib.mg_pack_weight_dgrad(_p(w_oihw), _p(wp), O, I, KH, KW, stride, k0h, Jh, k0w, Jw, _p(inv_sigma), _stream()),
                  "mg_pack_weight_dgrad")
            extra = dict(pad_h_extra=ph, pad_w_extra=pw, out_stride=stride, out_off_h=rh, out_off_w=rw, OHF=H, OWF=W,
                         accumulate=int(accumulate))
            if dy16 is not None:
                conv_igemm(dy16, cvt16(wp, BF16), I, Jh, Jw, 1, 0, out=out, out_hw=(ah, aw), _extra=extra, a_fmt=BF16)
            else:
                conv_igemm(dy, wp, I, Jh, Jw, 1, 0, out=out, out_hw=(ah, aw), _extra=extra)
    return out


def unpack_wgrad(dw_packed, shape_oihw, out=None, accumulate=False):
    O, I, KH, KW = shape_oihw
    if out is None:
        out = torch.empty(shape_oihw, device=dw_packed.device, dtype=torch.float32)
        accumulate = False
    check(_lib.load().mg_unpack_wgrad(_p(dw_packed), _p(out), O, I, KH, KW, int(accumulate), _stream()), "mg_unpack_wgrad")
    return out


def chan_sum(x):
    """Per-channel sum over all pixels of an NHWC tensor (bias gradients) -> [C] fp32."""
    return bn_sums(x)[: x.shape[-1]].float()


def spade_bwd(dh, h, g1, x, x_shift, nscale, nshift, act, dgb_fmt=TF32):
    """-> (dgb [N,H,W,2C] packed gamma|beta grads (fp32 TF32-rounded, or bf16 when dgb_fmt=BF16: the operand of the two
    gamma|beta gradient GEMMs), dxhat [N,H,W,C], sums [2C+1] float64, bias_sums [2C] float64 = per-channel sums of dgamma | dbeta)."""
    for t, nm in ((dh, "dh"), (h, "h"), (g1, "g1"), (x, "x")):
        _chk(t, nm)
    N, H, W, Cc = dh.shape
    dgb = torch.empty((N, H, W, 2 * Cc), device=dh.device, dtype=_dt(dgb_fmt))
    dxhat = torch.empty_like(dh)
    sums = torch.zeros(2 * Cc + 1, device=dh.device, dtype=torch.float64)   # + the sample-count slot (see bn_sums)
    bsums = torch.zeros(2 * Cc, device=dh.device, dtype=torch.float64)
    is16 = dgb_fmt != TF32
    check(_lib.load().mg_spade_bwd(_p(dh), _p(h), _p(g1), _p(x), x_shift, N, H, W, Cc, _p(nscale), _p(nshift), act, spade_bn(Cc),
                                   None if is16 else _p(dgb), _p(dxhat), _p(sums), _p(dgb) if is16 else None, _p(bsums), _stream()),
          "mg_spade_bwd")
    return dgb, dxhat, sums, bsums


def cvt16(x, fmt=BF16):
    """fp32 -> 16-bit copy (round to nearest) on the current stream."""
    _chk(x, "x")
    out = torch.empty(x.shape, device=x.device, dtype=_T16[fmt])
    check(_lib.load().mg_cvt16(_p(x), _p(out), x.numel(), fmt, _stream()), "mg_cvt16")
    return out


def conv_wgrad16(dy16, x16, kh, kw, stride=1, pad=0):
    """conv_wgrad with bf16 operands (fp32 accumulation and result)."""
    _chk(dy16, "dy16", torch.bfloat16); _chk(x16, "x16", torch.bfloat16)
    N, H, W, Cin = x16.shape
    _, OH, OW, Cout = dy16.shape
    dw = torch.empty((Cout, kh * kw * Cin), device=x16.device, dtype=torch.float32)
    check(_lib.load().mg_conv_wgrad16(_p(dy16), _p(x16), _p(dw), N, H, W, Cin, OH, OW, Cout, kh, kw, stride, pad, _stream()),
          "mg_conv_wgrad16")
    return dw


def bn_bwd_apply(g, x, x_shift, nscale, nshift, sums, count, dx=None):
    """dx (+)= BN backward of g through a folded 2^x_shift upsample (sums=None: plain child sum)."""
    _chk(g, "g"); _chk(x, "x"); _chk(dx, "dx")
    N, H, W, Cc = g.shape
    hs, ws = H >> x_shift, W >> x_shift
    acc = dx is not None
    if dx is None:
        dx = torch.empty((N, hs, ws, Cc), device=g.device, dtype=torch.float32)
    check(_lib.load().mg_bn_bwd_apply(_p(g), _p(x), x_shift, N, hs, ws, Cc, _p(nscale), _p(nshift), _p(sums), float(count), _p(dx),
                                      int(acc), _stream()), "mg_bn_bwd_apply")
    return dx


def blend_bwd(dout, hair, back, mask_stride, dbf=None):
    _chk(dout, "dout"); _chk(hair, "hair"); _chk(back, "back"); _chk(dbf, "dbf")
    N, H, W, Cc = dout.shape
    dy = torch.empty_like(dout)
    acc = dbf is not None
    if dbf is None:
        dbf = torch.empty_like(dout)
    check(_lib.load().mg_blend_bwd(_p(dout), _p(hair), _p(back), N, H, W, Cc, mask_stride, hair.shape[-2], hair.shape[-1], _p(dy),
                                   _p(dbf), int(acc), _stream()), "mg_blend_bwd")
    return dy, dbf


def act_bwd(dy, y, act, pm1=None, pm2=None, round_tf32=False):
    _chk(dy, "dy"); _chk(y, "y"); _chk(pm1, "pm1"); _chk(pm2, "pm2")
    Cc = dy.shape[-1]
    dz = torch.empty_like(dy)
    check(_lib.load().mg_act_bwd(_p(dy), _p(y), _p(dz), dy.numel() // Cc, Cc, act, _p(pm1), _p(pm2), int(round_tf32), _stream()),
          "mg_act_bwd")
    return dz


def maxpool2_relu_bwd(dpool, a, add=None, want_f32=True, want16=False):
    """Backward of y = maxpool2(relu output a): dx = [a > 0] * (pooled gradient routed to each window's arg-max + add).
    a: the saved tensor the forward pooled (fp32 or 16-bit); add: [N,H,W,C] fp32 or None.
    -> dx32, or (dx32|None, bf16 copy) with want16."""
    _chk(dpool, "dpool"); _chk(add, "add")
    a32, a16, afmt = _split32(a)
    N, H, W, Cc = a.shape
    assert tuple(dpool.shape) == (N, H // 2, W // 2, Cc), (dpool.shape, a.shape)
    dx = torch.empty((N, H, W, Cc), device=a.device, dtype=torch.float32) if want_f32 else None
    d16 = torch.empty((N, H, W, Cc), device=a.device, dtype=torch.bfloat16) if want16 else None
    check(_lib.load().mg_maxpool2_relu_bwd(_p(dpool), _p(a32), _p(a16), afmt, _p(add), _p(dx), _p(d16), N, H, W, Cc, _stream()),
          "mg_maxpool2_relu_bwd")
    if want16:
        return dx, d16
    return dx


def relu_bwd16(dy, a, add=None, want_f32=True, want16=False):
    """dz = [a > 0] * (dy + add) of an NHWC tensor (a fp32 or 16-bit).  -> dz32, or (dz32|None, bf16 copy) with want16."""
    _chk(dy, "dy"); _chk(add, "add")
    a32, a16, afmt = _split32(a)
    assert dy.shape == a.shape, (dy.shape, a.shape)
    dz = torch.empty(dy.shape, device=dy.device, dtype=torch.float32) if want_f32 else None
    d16 = torch.empty(dy.shape, device=dy.device, dtype=torch.bfloat16) if want16 else None
    check(_lib.load().mg_relu_bwd16(_p(dy), _p(add), _p(a32), _p(a16), afmt, _p(dz), _p(d16), dy.numel(), _stream()), "mg_relu_bwd16")
    if want16:
        return dz, d16
    return dz


def lab_loss_fwd(fake, real):
    """-> [1] float64 device tensor: sum over pixels of |a_fake - a_real| + |b_fake - b_real| (NCHW images in [-1, 1])."""
    _chk(fake, "fake"); _chk(real, "real")
    N, _, H, W = fake.shape
    assert fake.shape == real.shape and fake.shape[1] == 3, (fake.shape, real.shape)
    sums = torch.zeros(1, device=fake.device, dtype=torch.float64)
    check(_lib.load().mg_lab_loss_fwd(_p(fake), _p(real), _p(sums), N, H, W, _stream()), "mg_lab_loss_fwd")
    return sums


def lab_loss_bwd(fake, real, gscale):
    """d fake [N,3,H,W] of gscale[0] * lab_loss_fwd(fake, real); gscale: [1] fp32 device tensor."""
    _chk(fake, "fake"); _chk(real, "real"); _chk(gscale, "gscale")
    N, _, H, W = fake.shape
    dfake = torch.empty_like(fake)
    check(_lib.load().mg_lab_loss_bwd(_p(fake), _p(real), _p(gscale), _p(dfake), N, H, W, _stream()), "mg_lab_loss_bwd")
    return dfake


def hair_avg_lab_fwd(fake, real, mask_fake, mask_real):
    """-> [N,2,4] float64 device tensor: per image (sum m L, sum m a, sum m b, sum m) of fake with mask_fake, then of real with
    mask_real (NCHW images in [-1, 1], masks [N,1,H,W])."""
    _chk(fake, "fake"); _chk(real, "real"); _chk(mask_fake, "mask_fake"); _chk(mask_real, "mask_real")
    N, _, H, W = fake.shape
    assert fake.shape == real.shape and fake.shape[1] == 3, (fake.shape, real.shape)
    assert tuple(mask_fake.shape) == tuple(mask_real.shape) == (N, 1, H, W), (mask_fake.shape, mask_real.shape)
    sums = torch.empty((N, 2, 4), device=fake.device, dtype=torch.float64)
    check(_lib.load().mg_hair_avg_lab_fwd(_p(fake), _p(real), _p(mask_fake), _p(mask_real), _p(sums), N, H, W, _stream()),
          "mg_hair_avg_lab_fwd")
    return sums


def hair_avg_lab_bwd(fake, mask_fake, sums, g, out=None):
    """d fake [N,3,H,W] of g[0] * the hair-average Lab loss given hair_avg_lab_fwd's sums; g: [1] fp32 device tensor; out: a
    contiguous [N,3,H,W] fp32 tensor to write it into (default: a new one)."""
    _chk(fake, "fake"); _chk(mask_fake, "mask_fake"); _chk(sums, "sums", torch.float64); _chk(g, "g")
    N, _, H, W = fake.shape
    dfake = torch.empty_like(fake) if out is None else out
    if out is not None:
        _chk(out, "out")
        assert out.shape == fake.shape, (out.shape, fake.shape)
    check(_lib.load().mg_hair_avg_lab_bwd(_p(fake), _p(mask_fake), _p(sums), _p(g), _p(dfake), N, H, W, _stream()),
          "mg_hair_avg_lab_bwd")
    return dfake


class StyleTap(C.Structure):
    """One record of mg_style_loss_fwd's host table (include/michigan_b200.h); cnt_f / cnt_t set select the masked mode."""
    _fields_ = [("sums_f", C.c_void_p), ("sums_t", C.c_void_p), ("coef", C.c_void_p), ("M", C.c_longlong), ("N", C.c_int32),
                ("C", C.c_int32), ("cnt_f", C.c_void_p), ("cnt_t", C.c_void_p)]


def channel_sums(x):
    """Per-(image, channel) fp64 sums of an NHWC fp32 tensor -> [N, 2, C] (sum x, sum x^2), mg_in_stats."""
    _chk(x, "x")
    N, H, W, Cc = x.shape
    sums = torch.zeros((N, 2, Cc), device=x.device, dtype=torch.float64)
    check(_lib.load().mg_in_stats(_p(x), N, H * W, Cc, _p(sums), _stream()), "mg_in_stats")
    return sums


def style_loss_fwd(taps):
    """taps: list of (sums_fake [N,2,C], sums_target [N,2,C], M) -> ([1] float64 loss sum over the taps, [coef [N,3,C] per tap]).
    A tap (sums_fake, sums_target, M, cnt_fake [N], cnt_target [N]) takes the masked mode: the sums and the per-image mask
    counts of mg_loss_reduce op 10, the reference's calc_mean_std_mask, and coef is op 10's backward table.
    One mg_style_loss_fwd launch for every tap."""
    recs, coefs = [], []
    for tap in taps:
        sf, st, M = tap[:3]
        cf, ct = tap[3:] if len(tap) > 3 else (None, None)
        _chk(sf, "sums_f", torch.float64); _chk(st, "sums_t", torch.float64)
        _chk(cf, "cnt_f", torch.float64); _chk(ct, "cnt_t", torch.float64)
        N, _, Cc = sf.shape
        assert st.shape == sf.shape, (st.shape, sf.shape)
        assert cf is None or (cf.numel() == N and ct.numel() == N), (cf, ct)
        coef = torch.empty((N, 3, Cc), device=sf.device, dtype=torch.float32)
        coefs.append(coef)
        recs.append(StyleTap(_p(sf), _p(st), _p(coef), int(M), N, Cc, _p(cf), _p(ct)))
    loss = torch.zeros(1, device=taps[0][0].device, dtype=torch.float64)
    table = (StyleTap * len(recs))(*recs)
    check(_lib.load().mg_style_loss_fwd(C.cast(table, C.c_void_p), len(recs), _p(loss), _stream()), "mg_style_loss_fwd")
    return loss, coefs


def style_tap_grad(x, g, coef=None, content_t=None, add=None, out=None):
    """Gradient w.r.t. the fake tap x [N,h,w,C] of g[0] * style loss (coef from style_loss_fwd) + g[1] * content loss (MSE against
    content_t); g: [2] fp32 device tensor.  add (may be `out`) is accumulated; out defaults to a new tensor."""
    _chk(x, "x"); _chk(g, "g"); _chk(coef, "coef"); _chk(content_t, "content_t"); _chk(add, "add"); _chk(out, "out")
    N, H, W, Cc = x.shape
    if out is None:
        out = torch.empty_like(x)
    check(_lib.load().mg_style_tap_grad(_p(x), _p(coef), _p(content_t), _p(add), _p(out), _p(g), N, H * W, Cc, _stream()),
          "mg_style_tap_grad")
    return out


def pixel_l1_fwd(fake, tag, mask=None):
    """-> [1] float64 device tensor: sum |m*fake - m*tag| over [N,3,H,W] (mask [N,H,W] broadcast over channels; None = 1)."""
    _chk(fake, "fake"); _chk(tag, "tag"); _chk(mask, "mask")
    N, _, H, W = fake.shape
    assert fake.shape == tag.shape and fake.shape[1] == 3, (fake.shape, tag.shape)
    assert mask is None or tuple(mask.shape) == (N, H, W), mask.shape
    sums = torch.zeros(1, device=fake.device, dtype=torch.float64)
    check(_lib.load().mg_pixel_l1_fwd(_p(fake), _p(tag), _p(mask), _p(sums), N, H, W, _stream()), "mg_pixel_l1_fwd")
    return sums


def pixel_l1_bwd(fake, tag, gscale, mask=None):
    """d fake [N,3,H,W] of gscale[0] * pixel_l1_fwd(fake, tag, mask); gscale: [1] fp32 device tensor."""
    _chk(fake, "fake"); _chk(tag, "tag"); _chk(gscale, "gscale"); _chk(mask, "mask")
    N, _, H, W = fake.shape
    dfake = torch.empty_like(fake)
    check(_lib.load().mg_pixel_l1_bwd(_p(fake), _p(tag), _p(mask), _p(gscale), _p(dfake), N, H, W, _stream()), "mg_pixel_l1_bwd")
    return dfake


def instance_norm_act_fwd(x, act=ACT_LRELU, eps=1e-5, round_out=False, pmul=None, out16=None):
    """Training variant of instance_norm_act: also returns the (rstd, shift) table needed by in_bwd.
    -> (y, ss), or (y, ss, hi, lo|None) with out16=(fmt, want_lo) (16-bit operand copies for the next tensor-core conv)."""
    _chk(x, "x"); _chk(pmul, "pmul")
    N, H, W, Cc = x.shape
    sums = torch.zeros((N, 2, Cc), device=x.device, dtype=torch.float64)
    lib = _lib.load()
    check(lib.mg_in_stats(_p(x), N, H * W, Cc, _p(sums), _stream()), "mg_in_stats")
    ss = torch.empty((N, 2, Cc), device=x.device, dtype=torch.float32)
    y = torch.empty_like(x)
    hi, lo = _alloc16(tuple(x.shape), x.device, out16)
    check(lib.mg_in_apply(_p(x), _p(sums), _p(ss), _p(y), N, H * W, Cc, eps, act, int(round_out), _p(pmul), _p(hi), _p(lo),
                          (out16[0] if out16 else 0), _stream()), "mg_in_apply")
    if out16 is not None:
        return y, ss, hi, lo
    return y, ss


def in_bwd(df, x, ss, act=ACT_LRELU, pmul=None, round_tf32=False):
    _chk(df, "df"); _chk(x, "x"); _chk(ss, "ss"); _chk(pmul, "pmul")
    N, H, W, Cc = x.shape
    sums = torch.empty((N, 2, Cc), device=x.device, dtype=torch.float64)
    dx = torch.empty_like(x)
    check(_lib.load().mg_in_bwd(_p(df), _p(x), _p(ss), _p(sums), _p(dx), N, H * W, Cc, act, _p(pmul), int(round_tf32), _stream()),
          "mg_in_bwd")
    return dx


def thin_wgrad(x, dz, kh, kw, stride, pad, pad_mode=0, seg_resize=0, in_hw=None, relu_src=None, want_bias=False):
    """dwt [kh*kw][CinP][Cout] of a thin conv; x is the (possibly full-resolution seg) input.
    Register-tiled CUDA-core kernel (4 output channels x <= 13 weight columns per thread).
    relu_src: the conv's forward output y - dz is multiplied by [y > 0] on the fly (ReLU backward fused in);
    want_bias: also return the per-channel sums of that dz (the bias gradient) -> (dwt, bias[Cout] fp32)."""
    _chk(x, "x"); _chk(dz, "dz"); _chk(relu_src, "relu_src")
    N, OH, OW, Cout = dz.shape
    CinP = x.shape[-1]
    H, W = in_hw if seg_resize else (x.shape[1], x.shape[2])
    dwt = torch.empty((kh * kw, CinP, Cout), device=x.device, dtype=torch.float32)
    bsum = torch.zeros(Cout, device=x.device, dtype=torch.float64) if want_bias else None
    check(_lib.load().mg_thin_wgrad(_p(x), _p(dz), _p(dwt), N, H, W, CinP, OH, OW, Cout, kh, kw, stride, pad, pad_mode, seg_resize,
                                    _p(relu_src), _p(bsum), _stream()), "mg_thin_wgrad")
    if want_bias:
        return dwt, bsum.float()
    return dwt


def thin_dgrad3(dz, wt, dimg_nchw, kh, kw, stride, pad, c_lo):
    _chk(dz, "dz"); _chk(wt, "wt"); _chk(dimg_nchw, "dimg")
    N, OH, OW, Cout = dz.shape
    _, _, H, W = dimg_nchw.shape
    check(_lib.load().mg_thin_dgrad3(_p(dz), _p(wt), _p(dimg_nchw), N, H, W, wt.shape[1], OH, OW, Cout, kh, kw, stride, pad, c_lo,
                                     _stream()), "mg_thin_dgrad3")
    return dimg_nchw


def conv_img_bwd(dy_nchw, y_nchw, x, w_oihw, act_in=ACT_LRELU, act_out=ACT_TANH):
    """-> (dx [N,H,W,Cin], dw [Cout,Cin,3,3], db [Cout])."""
    for t, nm in ((dy_nchw, "dy"), (y_nchw, "y"), (x, "x"), (w_oihw, "w")):
        _chk(t, nm)
    N, H, W, Cin = x.shape
    cout = w_oihw.shape[0]
    ws = torch.empty((N, H, W, 4), device=x.device, dtype=torch.float32)
    dx = torch.empty_like(x)
    dw = torch.zeros_like(w_oihw)
    db = torch.zeros(cout, device=x.device, dtype=torch.float32)
    check(_lib.load().mg_conv_img_bwd(_p(dy_nchw), _p(y_nchw), _p(x), _p(w_oihw), _p(ws), _p(dx), _p(dw), _p(db), N, H, W, Cin, cout,
                                      act_in, act_out, _stream()), "mg_conv_img_bwd")
    return dx, dw, db


def conv_to1_bwd(dl, x, w_oihw, pad, dx=None, want_dx=True):
    """-> (dx (+= when given), dw, db) of the Cin->1 logits conv."""
    _chk(dl, "dl"); _chk(x, "x"); _chk(w_oihw, "w"); _chk(dx, "dx")
    N, H, W, Cin = x.shape
    _, _, KH, KW = w_oihw.shape
    acc = dx is not None
    if dx is None and want_dx:
        dx = torch.empty_like(x)
    dw = torch.zeros_like(w_oihw)
    db = torch.zeros(1, device=x.device, dtype=torch.float32)
    check(_lib.load().mg_conv_to1_bwd(_p(dl), _p(x), _p(w_oihw), _p(dx), _p(dw), _p(db), N, H, W, Cin, KH, KW, pad, int(acc), _stream()),
          "mg_conv_to1_bwd")
    return dx, dw, db


def avgpool3s2_bwd(dout, din_accum):
    _chk(dout, "dout"); _chk(din_accum, "din")
    N, H, W, Cc = din_accum.shape
    check(_lib.load().mg_avgpool3s2_bwd(_p(dout), _p(din_accum), N, H, W, Cc, dout.shape[1], dout.shape[2], _stream()),
          "mg_avgpool3s2_bwd")
    return din_accum


def reflect_pad_bwd(dpad, pad, dx=None):
    _chk(dpad, "dpad"); _chk(dx, "dx")
    N, PH, PW, Cc = dpad.shape
    H, W = PH - 2 * pad, PW - 2 * pad
    acc = dx is not None
    if dx is None:
        dx = torch.empty((N, H, W, Cc), device=dpad.device, dtype=torch.float32)
    check(_lib.load().mg_reflect_pad_bwd(_p(dpad), _p(dx), N, H, W, Cc, pad, int(acc), _stream()), "mg_reflect_pad_bwd")
    return dx


def resize_bilinear_bwd(dout, in_hw):
    _chk(dout, "dout")
    N, OH, OW, Cc = dout.shape
    din = torch.zeros((N, in_hw[0], in_hw[1], Cc), device=dout.device, dtype=torch.float32)
    check(_lib.load().mg_resize_bilinear_bwd(_p(dout), _p(din), N, in_hw[0], in_hw[1], Cc, OH, OW, _stream()), "mg_resize_bilinear_bwd")
    return din


def masked_mean_bcast_bwd(dout, mref, mtag):
    """Gradient of masked_mean_bcast w.r.t. x, with the same None modes."""
    _chk(dout, "dout"); _chk(mref, "mref"); _chk(mtag, "mtag")
    N, h, w, Cc = dout.shape
    MH, MW = _mask_hw(mref, mtag, h, w)
    dx = torch.empty_like(dout)
    check(_lib.load().mg_masked_mean_bcast_bwd(_p(dout), _p(mref), _p(mtag), _p(dx), N, h, w, Cc, MH, MW, _stream()),
          "mg_masked_mean_bcast_bwd")
    return dx


def spectral_norm_bwd(dwt_oihw, w_orig, u, v, inv_sigma, out=None):
    """Gradient w.r.t. weight_orig given the gradient w.r.t. W/sigma (u, v treated as constants)."""
    for t, nm in ((dwt_oihw, "dwt"), (w_orig, "w_orig"), (u, "u"), (v, "v"), (inv_sigma, "inv_sigma")):
        _chk(t, nm)
    O = w_orig.shape[0]
    K = w_orig[0].numel()
    acc = out is not None
    if out is None:
        out = torch.empty_like(w_orig)
    dot = torch.empty(1, device=w_orig.device, dtype=torch.float64)
    check(_lib.load().mg_spectral_norm_bwd(_p(dwt_oihw), _p(w_orig), _p(u), _p(v), _p(inv_sigma), _p(dot), _p(out), O, K, int(acc),
                                           _stream()), "mg_spectral_norm_bwd")
    return out


def pack_weight_dgrad_gb(wg, wb):
    _chk(wg, "wg"); _chk(wb, "wb")
    Cc, I, _, _ = wg.shape
    out = torch.empty((I, 9 * 2 * Cc), device=wg.device, dtype=torch.float32)
    check(_lib.load().mg_pack_weight_dgrad_gb(_p(wg), _p(wb), _p(out), Cc, I, spade_bn(Cc), _stream()), "mg_pack_weight_dgrad_gb")
    return out


def unpack_wgrad_gb(dw_packed, c, i):
    _chk(dw_packed, "dw_packed")
    dwg = torch.empty((c, i, 3, 3), device=dw_packed.device, dtype=torch.float32)
    dwb = torch.empty_like(dwg)
    check(_lib.load().mg_unpack_wgrad_gb(_p(dw_packed), _p(dwg), _p(dwb), c, i, spade_bn(c), 0, _stream()), "mg_unpack_wgrad_gb")
    return dwg, dwb
