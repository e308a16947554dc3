"""ctypes binding of libmichigan_sm90.so (C ABI declared in include/michigan_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, an exception is
raised.  The product path never routes through PyTorch eager or the CPU oracle.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# MICHIGAN_B200_LIB: tools/ select the -DMG_PROBES build (timing experiments); the product always loads the in-tree release library
LIB_PATH = os.environ.get("MICHIGAN_B200_LIB") or os.path.join(_HERE, "lib", "libmichigan_sm90.so")

c_f32p = C.c_void_p  # device pointers travel as integers (tensor.data_ptr())


class IgemmArgs(C.Structure):
    _fields_ = [
        ("inp", c_f32p), ("wpack", c_f32p), ("out", c_f32p),
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cin", C.c_int32),
        ("OH", C.c_int32), ("OW", C.c_int32), ("Cout", C.c_int32),
        ("KH", C.c_int32), ("KW", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("BN", C.c_int32),
        ("epi", C.c_int32), ("act", C.c_int32), ("round_out", C.c_int32),
        ("bias", c_f32p), ("res", c_f32p), ("res_shift", C.c_int32),
        ("pscale", c_f32p), ("pmul", c_f32p),
        ("bf", c_f32p), ("hair", c_f32p), ("back", c_f32p),
        ("mask_stride", C.c_int32), ("MH", C.c_int32), ("MW", C.c_int32),
        ("x", c_f32p), ("x_shift", C.c_int32),
        ("nscale", c_f32p), ("nshift", c_f32p), ("gbias1", c_f32p), ("bbias", c_f32p),
        ("max_ctas", C.c_int32),
        ("pad_h_extra", C.c_int32), ("pad_w_extra", C.c_int32),
        ("out_stride", C.c_int32), ("out_off_h", C.c_int32), ("out_off_w", C.c_int32),
        ("OHF", C.c_int32), ("OWF", C.c_int32), ("accumulate", C.c_int32),
        ("in_lo", c_f32p), ("a_fmt", C.c_int32), ("split", C.c_int32),
        ("out_hi", c_f32p), ("out_lo", c_f32p), ("out16_fmt", C.c_int32),
        ("aux_out", c_f32p),
    ]


class ThinArgs(C.Structure):
    _fields_ = [
        ("inp", c_f32p), ("w", c_f32p), ("bias", c_f32p), ("out", c_f32p),
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("CinP", C.c_int32),
        ("OH", C.c_int32), ("OW", C.c_int32), ("Cout", C.c_int32),
        ("KH", C.c_int32), ("KW", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("pad_mode", C.c_int32), ("seg_resize", C.c_int32),
        ("act", C.c_int32), ("round_out", C.c_int32),
        ("pscale", c_f32p), ("pmul", c_f32p),
        ("out_hi", c_f32p), ("out_lo", c_f32p), ("out16_fmt", C.c_int32),
    ]


_i, _ll, _f, _d, _p = C.c_int, C.c_longlong, C.c_float, C.c_double, C.c_void_p

# name -> argtypes (all return int unless noted); mirrors include/michigan_b200.h
SIGNATURES = {
    "mg_version": [],
    "mg_last_error": [],
    "mg_launch_count": [],
    "mg_set_tuning": [C.c_char_p, _i],
    "mg_get_tuning": [C.c_char_p],
    "mg_conv_igemm": [C.POINTER(IgemmArgs), _p],
    "mg_pack_weight": [_p, _p, _i, _i, _i, _i, _p, _i, _p],
    "mg_pack_weight_gb": [_p, _p, _p, _i, _i, _i, _i, _i, _p],
    "mg_pack_weight16": [_p, _p, _i, _i, _i, _i, _p, _i, _i, _p],
    "mg_pack_weight_gb16": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_conv_thin": [C.POINTER(ThinArgs), _p],
    "mg_pack_weight_thin": [_p, _p, _i, _i, _i, _i, _i, _p],
    "mg_conv_seg_tc": [C.POINTER(ThinArgs), _p],
    "mg_pack_weight_seg_tc": [_p, _p, _i, _i, _p],
    "mg_debug_seg_prof": [C.c_void_p],
    "mg_conv_img": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_conv_to1": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_bn_stats": [_p, _ll, _i, _p, _p],
    "mg_bn_stats_cvt16": [_p, _ll, _i, _p, _p, _p],
    "mg_bn_finalize": [_p, _i, _d, _d, _f, _f, _i, _p, _p, _p, _p, _p, _p, _p],
    "mg_bn_from_running": [_p, _p, _i, _f, _p, _p, _p],
    "mg_in_stats": [_p, _i, _ll, _i, _p, _p],
    "mg_in_apply": [_p, _p, _p, _p, _i, _ll, _i, _f, _i, _i, _p, _p, _p, _i, _p],
    "mg_prep_seg": [_p, _p, _i, _p, _i, _i, _i, _p],
    "mg_prep_dinput": [_p, _p, _p, _i, _i, _i, _p],
    "mg_prep_bginput": [_p, _p, _p, _p, _i, _i, _i, _p],
    "mg_nchw_to_nhwc": [_p, _p, _i, _i, _i, _i, _i, _p, _p],
    "mg_partial_mask": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_masked_mean_bcast": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_resize_bilinear": [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_reflect_pad": [_p, _p, _i, _i, _i, _i, _i, _i, _p, _p, _i, _p],
    "mg_spectral_norm_batched": [_p, _i, _i, _i, _i, _f, _p],
    "mg_pack_weight_dgrad": [_p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p],
    "mg_unpack_wgrad": [_p, _p, _i, _i, _i, _i, _i, _p],
    "mg_conv_wgrad": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_spade_bwd": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p, _i, _i, _p, _p, _p, _p, _p, _p],
    "mg_cvt16": [_p, _p, _ll, _i, _p],
    "mg_conv_wgrad16": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_bn_bwd_apply": [_p, _p, _i, _i, _i, _i, _i, _p, _p, _p, _d, _p, _i, _p],
    "mg_blend_bwd": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _i, _p],
    "mg_act_bwd": [_p, _p, _p, _ll, _i, _i, _p, _p, _i, _p],
    "mg_in_bwd": [_p, _p, _p, _p, _p, _i, _ll, _i, _i, _p, _i, _p],
    "mg_thin_wgrad": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p],
    "mg_thin_dgrad3": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_conv_img_bwd": [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_conv_to1_bwd": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p],
    "mg_avgpool3s2_bwd": [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_reflect_pad_bwd": [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_resize_bilinear_bwd": [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_masked_mean_bcast_bwd": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_spectral_norm_bwd": [_p, _p, _p, _p, _p, _p, _p, _i, _ll, _i, _p],
    "mg_pack_weight_dgrad_gb": [_p, _p, _p, _i, _i, _i, _p],
    "mg_unpack_wgrad_gb": [_p, _p, _p, _i, _i, _i, _i, _p],
    "mg_nhwc_to_nchw": [_p, _p, _i, _i, _i, _i, _i, _p],
    "mg_maxpool_mask": [_p, _p, _p, _i, _i, _i, _i, _i, _p],
    "mg_avgpool3s2": [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    "mg_softmax_rows": [_p, _ll, _i, _p, _p, _p, _i, _i, _p],
    "mg_noise_pyramid": [_p, _i, _p, _i, _i, _i, _p],
    "mg_orient_rgb": [_p, _p, _p, _i, _i, _i, _p],
    "mg_hole_mask": [_p, _p, _p, _p, _p, _i, _i, _i, _p],
    "mg_orient_loss_fwd": [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "mg_orient_loss_bwd": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "mg_edge_weight": [_p, _p, _i, _i, _i, _i, _i, _f, _p],
    "mg_loss_reduce": [_p, _i, _p, _p],
    "mg_loss_reduce_bwd": [_p, _i, _p, _p],
    "mg_loss_term_bytes": [],
    "mg_maxpool2_nhwc": [_p, _p, _i, _p, _p, _i, _i, _i, _i, _i, _p],
    "mg_maxpool2_relu_bwd": [_p, _p, _p, _i, _p, _p, _p, _i, _i, _i, _i, _p],
    "mg_relu_bwd16": [_p, _p, _p, _p, _i, _p, _p, _ll, _p],
    "mg_lab_loss_fwd": [_p, _p, _p, _i, _i, _i, _p],
    "mg_lab_loss_bwd": [_p, _p, _p, _p, _i, _i, _i, _p],
    "mg_hair_avg_lab_fwd": [_p, _p, _p, _p, _p, _i, _i, _i, _p],
    "mg_hair_avg_lab_bwd": [_p, _p, _p, _p, _p, _i, _i, _i, _p],
    "mg_style_loss_fwd": [_p, _i, _p, _p],
    "mg_style_tap_bytes": [],
    "mg_style_tap_grad": [_p, _p, _p, _p, _p, _p, _i, _ll, _i, _p],
    "mg_pixel_l1_fwd": [_p, _p, _p, _p, _i, _i, _i, _p],
    "mg_pixel_l1_bwd": [_p, _p, _p, _p, _p, _i, _i, _i, _p],
    "mg_peer_buffer_bytes": [_i],
    "mg_peer_max_elems": [],
    "mg_peer_allreduce_f64": [_p, _i, _p, _i, _i, C.c_ulonglong, _i, _d, _p, _p],
}

_lib = None


class MichiganNativeError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises if it has not been built: there is no CPU fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MichiganNativeError(
            "libmichigan_sm90.so not found at %s - run `python -m michigan_b200.build` "
            "(the CUDA extension is mandatory; there is no fallback path)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.mg_last_error.restype = C.c_char_p
    lib.mg_launch_count.restype = C.c_longlong
    lib.mg_peer_buffer_bytes.restype = C.c_longlong
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().mg_last_error().decode("utf-8", "replace")
        raise MichiganNativeError("%s failed (status %d): %s" % (what or "libmichigan_sm90 call", rc, msg))


def set_tuning(name, value):
    """Schedule knob of the library (see mg_set_tuning in the header); returns the previous value."""
    lib = load()
    prev = lib.mg_get_tuning(name.encode())
    check(lib.mg_set_tuning(name.encode(), int(value)), "mg_set_tuning")
    return prev


def launch_count():
    return int(load().mg_launch_count())
