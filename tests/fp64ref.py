"""Float64 reference helpers shared by the GPU tests that hold CUDA results to fp64 CPU autograd element by element:

    |got - ref| <= k * u * R_abs + TINY

R_abs is the magnitude reference: the same fp64 computation on |inputs|; u the unit roundoff of the coarsest operand format
involved; k a measured constant with headroom.
"""
import torch

U = 2.0 ** -24        # fp32 unit roundoff
U_TF32 = 2.0 ** -11   # TF32 and fp16 operands (11 significand bits)
U_BF16 = 2.0 ** -8    # one-pass bf16 operands
TINY = 1e-30


def tf32_trunc(t):
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def rna_tf32(t):
    """cvt.rna.tf32.f32 on finite fp32 values: round the magnitude to 10 stored mantissa bits, ties away from zero."""
    return ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def d64(t):
    return t.detach().cpu().double()


def vjp64(fn, inputs, dout):
    """fp64 CPU autograd: -> (fn(*inputs), d inputs) for the output gradient dout."""
    xs = [d64(t).requires_grad_(True) for t in inputs]
    out = fn(*xs)
    gs = torch.autograd.grad(out, xs, d64(dout), allow_unused=True)
    return out.detach(), gs


def check_close(name, got, ref, rabs, k, u=U, skip=None):
    """|got - ref| <= k * u * rabs + TINY for every element (skip: boolean mask of elements left out).  Returns the largest
    measured |got - ref| / (u * rabs)."""
    got, ref, rabs = d64(got), d64(ref), d64(rabs)
    assert got.shape == ref.shape == rabs.shape, (name, got.shape, ref.shape, rabs.shape)
    assert bool(torch.isfinite(got).all()), name
    err = (got - ref).abs()
    if skip is not None:
        err = torch.where(skip, torch.zeros_like(err), err)
    ratio = float((err / (u * rabs + TINY)).max())
    print("%s: max |got - ref| / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > k * u * rabs + TINY
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements out of bound; max ratio %.3g > k = %g; first at %s: got %r ref %r R_abs %r"
                             % (name, int(bad.sum()), bad.numel(), ratio, k, i, float(got[i]), float(ref[i]), float(rabs[i])))
    return ratio
