"""The 3x3 M-tile-group kernel (mg_conv3x3.cu) has two epilogues: straight from the wgmma accumulator registers
(MG_EPI_REG=1, the default) and through a shared-memory accumulator tile (MG_EPI_REG=0).  They run the same per-element
arithmetic on the same accumulators, so every output (fp32, 16-bit hi/lo, the SPADE 1 + gamma copy) must be bit-identical.
The plain epilogue at BN = 128 without merged halves takes the staged path under both settings (conv3_reg_epilogue).
Shapes are small but eligible for the group kernel (OW % 16 == 0, OH >= 16); OH = 40 leaves a partial 16-row tile, and
max_ctas = 5 gives every CTA several groups."""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"

# operand format -> (a_fmt, split)
FMTS = {"tf32": (0, False), "f16": (1, False), "bf16": (2, False), "f16_split": (1, True), "bf16_split": (2, True)}


def _lib_mod():
    from michigan_b200 import _lib
    return _lib


def _ops():
    from michigan_b200 import ops
    return ops


def _operands(ops, x, fmt):
    """x [N,H,W,C] fp32 -> (operand, operand_lo | None) in the kernel's input format."""
    a_fmt, split = FMTS[fmt]
    if a_fmt == ops.TF32:
        return (x.view(torch.int32) & ~0x1FFF).view(torch.float32), None
    t = torch.float16 if a_fmt == ops.F16 else torch.bfloat16
    hi = x.to(t)
    return hi, ((x - hi.float()).to(t) if split else None)


def _both(run):
    """run() under MG_EPI_REG = 1 and 0 -> two lists of output tensors."""
    outs = {}
    for reg in (1, 0):
        prev = _lib_mod().set_tuning("MG_EPI_REG", reg)
        try:
            outs[reg] = [t.clone() for t in run() if t is not None]
            torch.cuda.synchronize()
        finally:
            _lib_mod().set_tuning("MG_EPI_REG", prev)
    return outs[1], outs[0]


def _assert_equal(new, old):
    assert len(new) == len(old) and new
    for i, (a, b) in enumerate(zip(new, old)):
        assert torch.isfinite(a.float()).all(), i
        assert torch.equal(a, b), (i, float((a.float() - b.float()).abs().max()))


PLAIN = [
    # fmt, Cout, bn, h, w, features
    ("tf32", 64, 0, 32, 48, {"bias", "res"}),
    ("tf32", 128, 64, 40, 48, {"bias", "res1", "round"}),
    ("f16", 128, 128, 32, 48, {"bias", "res", "out16"}),
    ("bf16", 64, 0, 40, 32, {"pscale", "pmul", "accumulate"}),
    ("f16_split", 64, 0, 32, 48, {"bias", "blend"}),
    ("bf16_split", 64, 0, 40, 48, {"bias", "res", "out16"}),     # merged (2 BN <= 128)
    ("bf16_split", 128, 64, 32, 32, {"bias", "res1", "pmul"}),   # merged at BN 64
    ("bf16_split", 256, 0, 40, 48, {"bias", "res", "out16"}),    # 3-pass (BN 128)
    ("f16", 64, 0, 40, 48, {"blend2", "accumulate", "round"}),
]


@pytest.mark.parametrize("fmt,Cout,bn,h,w,feat", PLAIN)
def test_reg_epilogue_plain_bitwise(fmt, Cout, bn, h, w, feat):
    ops = _ops()
    g = torch.Generator(device="cpu").manual_seed(7)
    N, Cin = 2, 128
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    x, x_lo = _operands(ops, r(N, h, w, Cin), fmt)
    wt = r(Cout, Cin, 3, 3) / (3 * Cin ** 0.5)
    a_fmt, split = FMTS[fmt]
    wp = ops.pack_weight(wt, None, round_tf32=True) if a_fmt == ops.TF32 else ops.pack_weight16(wt, None, a_fmt, split=split)
    kw = dict(act=2, a_fmt=a_fmt, x_lo=x_lo, bn=bn, max_ctas=5)
    if "bias" in feat:
        kw["bias"] = r(Cout)
    if "res" in feat:
        kw["res"] = r(N, h, w, Cout)
    if "res1" in feat:
        kw["res"], kw["res_shift"] = r(N, h // 2, w // 2, Cout), 1
    if "pscale" in feat:
        kw["pscale"] = torch.rand(N, h, w, generator=g).to(dev) + 0.5
    if "pmul" in feat:
        kw["pmul"] = torch.rand(N, h, w, generator=g).to(dev)
    if "blend" in feat or "blend2" in feat:
        ms = 2 if "blend2" in feat else 1
        kw["blend"] = (r(N, h, w, Cout), torch.rand(N, h * ms, w * ms, generator=g).to(dev),
                       torch.rand(N, h * ms, w * ms, generator=g).to(dev), ms)
    if "round" in feat:
        kw["round_out"] = True
    if "out16" in feat:
        kw["out16"] = (ops.BF16 if fmt != "f16" else ops.F16, True)
    init = r(N, h, w, Cout)

    def run():
        out = init.clone() if "accumulate" in feat else torch.full_like(init, float("nan"))
        res = ops.conv_igemm(x, wp, Cout, 3, 3, 1, 1, out=out, _extra={"accumulate": int("accumulate" in feat)}, **kw)
        return list(res) if isinstance(res, tuple) else [res]

    _assert_equal(*_both(run))


SPADE = [
    # fmt, C (BN = 64 for C = 32, else 128), h, w, x_shift, act, mode
    ("f16", 64, 32, 48, 1, 2, "spec"),       # SPEC 1: lrelu -> bf16 hi/lo only
    ("f16", 128, 40, 48, 0, 0, "spec"),      # SPEC 2: no activation, two N tiles, partial row tile
    ("tf32", 32, 32, 48, 0, 2, "spec"),      # BN 64
    ("bf16_split", 32, 40, 32, 1, 2, "spec"),  # merged split precision, SPADE
    ("tf32", 64, 32, 48, 1, 2, "aux"),       # SPEC 0: fp32 out + 1 + gamma (training)
    ("f16", 32, 40, 48, 0, 0, "aux"),
    ("bf16_split", 32, 32, 48, 0, 2, "aux"),
]


@pytest.mark.parametrize("fmt,C,h,w,xs,act,mode", SPADE)
def test_reg_epilogue_spade_bitwise(fmt, C, h, w, xs, act, mode):
    ops = _ops()
    g = torch.Generator(device="cpu").manual_seed(11)
    N, Cin = 2, 128
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    actv, a_lo = _operands(ops, r(N, h, w, Cin), fmt)
    wg, wb = r(C, Cin, 3, 3) / 34, r(C, Cin, 3, 3) / 34
    a_fmt, split = FMTS[fmt]
    wp = ops.pack_weight_gb(wg, wb) if a_fmt == ops.TF32 else ops.pack_weight_gb16(wg, wb, a_fmt, split=split)
    spade = (r(N, h >> xs, w >> xs, C), xs, r(C), r(C), r(C), r(C))

    def run():
        if mode == "spec":
            return list(ops.conv_igemm(actv, wp, C, 3, 3, 1, 1, act=act, a_fmt=a_fmt, x_lo=a_lo, spade=spade,
                                       out16=(ops.BF16, True), want_f32=False, max_ctas=5))
        aux = torch.full((N, h, w, C), float("nan"), device=dev)
        out = ops.conv_igemm(actv, wp, C, 3, 3, 1, 1, act=act, a_fmt=a_fmt, x_lo=a_lo, spade=spade, aux=aux, max_ctas=5)
        return [out, aux]

    _assert_equal(*_both(run))
