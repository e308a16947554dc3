"""GAN loss and GAN feature-matching loss with the reference's call signatures
(models/networks/loss.py:19-140 `GANLoss`, every gan_mode ('ls', 'original', 'w', 'hinge'), 144-175 `GANFeatLoss`, with and
without --remove_background), evaluated by the fused reduction kernels of csrc/mg_loss.cu:

  * every call = ONE forward launch (all discriminator scales / all eight feature terms through a descriptor table,
    fp64 accumulation) and ONE backward launch, instead of ~10 eager ops per scale and per term;
  * the wide-edge weight map (loss.py:60-78) is one kernel per scale, cached per (label, size) within an iteration.

The rest of the generator objective follows: the Gabor and DoG orientation losses, VGGLoss / StyleContentLoss (every VGG19 term from one
pass, _VGGObjectiveFn), LabColorLoss and HairAvgLabLoss (with or without --balance_Lab), RGBBackgroundL1Loss and the rgb L1
(RGBL1Loss), and the --use_vae KLDLoss.
"""
import ctypes as C
import os
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib, ops


class _Term(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("ga", C.c_void_p), ("n", C.c_longlong), ("scale", C.c_float),
                ("sign", C.c_float), ("op", C.c_int32), ("out_slot", C.c_int32),
                # appended for ops 4-8 (zero for ops 0-3)
                ("target", C.c_float), ("den_slot", C.c_int32), ("label", C.c_void_p), ("label_ns", C.c_longlong),
                ("C", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("channels_last", C.c_int32),
                # appended for the accumulating backward (null: ga is written, not accumulated)
                ("add", C.c_void_p),
                # appended for op 11 (null for every other op)
                ("table", C.c_void_p),
                # appended for op 12 (null for every other op)
                ("idx", C.c_void_p), ("maxv", C.c_void_p)]


OP_HINGE_D, OP_SUM, OP_L1, OP_SQ = 0, 1, 2, 3
# gan_mode 'original' / 'ls' against a constant target; the --remove_background terms, masked by the resized hair label
OP_BCE, OP_SQ_T, OP_WSUM, OP_HINGE_MASK, OP_L1_MASK = 4, 5, 6, 7, 8
# --remove_background in VGGLoss / StyleContentLoss: the masked content term and the masked channel moments of one VGG tap
OP_SQ_MASK, OP_MOMENTS = 9, 10
# LabColorLoss with --balance_Lab: the Lab L1 weighted per pixel by the count table of the real pixel's (a, b) bins
OP_LAB_BALANCED = 11
# L1OLoss with the DoG filter: both losses of the batch-normalised confidence and the sums of the gradient through its maximum
OP_ORIENT_DOG = 12
# KLDLoss: the logvar half, e^a - a - 1 (the mu half is OP_SQ against zeros)
OP_KLD_EXP = 13
MASKED_OPS = (OP_WSUM, OP_HINGE_MASK, OP_L1_MASK, OP_SQ_MASK)      # one scalar term over its own sum(label1) * c + 1e-5
DEN_EPS = 1e-5          # loss.py:111, 114, 117, 160, 196, 677: sum(label1) * c + 1e-5
_table_cache = {}


class _Spec(namedtuple("_Spec", "op ai b scale sign slot target label")):
    """One loss term: op, index of its differentiable input `a`, the detached `b` (or None), scale, hinge sign, output slot;
    the constant target of ops 4 and 5; the [N,1,H,W] hair label of the masked ops."""
    __slots__ = ()

    def __new__(cls, op, ai, b, scale, sign, slot, target=0.0, label=None):
        return super().__new__(cls, op, ai, b, scale, sign, slot, target, label)


def _dense(t):
    """A tensor whose elements occupy one contiguous block (any permutation of strides) or a contiguous copy."""
    if t.is_contiguous() or (t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)):
        return t
    return t.contiguous()


def _hair_label(label, x):
    """The [N,1,H,W] label the masked terms of x ([N,C,h,w]) read in place: fp32, rows contiguous, any image stride (the hair
    channel of the one-hot label map is a view)."""
    if label is None:
        raise ValueError("--remove_background needs the hair label")
    lab = label.detach()
    if lab.dim() != 4 or lab.shape[1] != 1 or lab.shape[0] != x.shape[0] or x.dim() != 4:
        raise ValueError("--remove_background: label %s does not match the [N,C,h,w] input %s" % (tuple(lab.shape), tuple(x.shape)))
    lab = lab.float()
    _, _, H, W = lab.shape
    if not ((W == 1 or lab.stride(3) == 1) and (H == 1 or lab.stride(2) == W)):
        lab = lab.contiguous()
    return lab


def _device_table(terms, device):
    """ctypes term records -> device buffer (cached: the caching allocator hands the same addresses back every iteration)."""
    raw = bytes((_Term * len(terms))(*terms))
    hit = _table_cache.get(raw)
    if hit is not None and hit.device == device:
        return hit
    if len(_table_cache) > 256:
        _table_cache.clear()
    buf = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)
    _table_cache[raw] = buf
    return buf


def _fold_masked(nums, dens):
    """The masked terms' values sum_k nums[k] / (dens[k] + 1e-5), formed on the device (no host synchronisation), and the
    1 / (dens + 1e-5) that scale their gradients (_masked_gslots)."""
    inv = 1.0 / (dens + DEN_EPS)
    return (nums * inv).sum(), inv


def _masked_gslots(g, inv):
    """The gradient slots of masked terms: the upstream gradient g over each term's denominator, fp32."""
    return (g.double() * inv).float()


def _term(s, a, b, ga, out_slot, den_slot, add=None):
    """The _Term record of spec s on a ([N,C,h,w], NCHW or channels-last for the masked ops); ga, add: gradient pointers."""
    t = _Term(a.data_ptr(), b.data_ptr() if b is not None else None, ga, a.numel(), float(s.scale), float(s.sign), s.op, out_slot)
    t.target = float(s.target)
    t.add = add
    if s.op in MASKED_OPS or s.op == OP_MOMENTS:
        lab = s.label
        t.den_slot, t.label, t.label_ns = den_slot, lab.data_ptr(), lab.stride(0)
        t.C, t.h, t.w = a.shape[1], a.shape[2], a.shape[3]
        t.H, t.W = lab.shape[2], lab.shape[3]
        t.channels_last = int(not a.is_contiguous())
    return t


class _LossFn(torch.autograd.Function):
    """spec: list of _Spec (or of their first six fields as a tuple); tensors: the differentiable `a` inputs.  A masked term k (ops 6-8) sums into a slot of its own,
    nslots + k', and its label sum into nslots + m + k' (m masked terms); its slot then adds num / (den + 1e-5) on the
    device, and its gradient is scaled by the same 1 / (den + 1e-5)."""

    @staticmethod
    def forward(ctx, spec, nslots, *tensors):
        assert _lib.load().mg_loss_term_bytes() == C.sizeof(_Term)
        spec = [s if isinstance(s, _Spec) else _Spec(*s) for s in spec]        # plain (op, ai, b, scale, sign, slot) tuples too
        dense = [_dense(t.detach()) for t in tensors]
        dev = dense[0].device
        masked = [k for k, s in enumerate(spec) if s.op in MASKED_OPS]
        m = len(masked)
        if m and len({spec[k].slot for k in masked}) != 1:
            raise ValueError("the masked terms of one loss add into one slot")
        terms = []
        keep = []
        slot_of = {}
        for k, s in enumerate(spec):
            a = dense[s.ai]
            bb = _dense(s.b.detach()) if s.b is not None else None
            if bb is not None:
                assert bb.numel() == a.numel(), (bb.shape, a.shape)
                if s.op == OP_L1_MASK:
                    assert bb.shape == a.shape and bb.stride() == a.stride(), (bb.shape, bb.stride(), a.shape, a.stride())
                keep.append(bb)
            out_slot, den_slot = s.slot, 0
            if s.op in MASKED_OPS:
                j = masked.index(k)
                out_slot, den_slot = nslots + j, nslots + m + j
                assert a.dim() == 4 and s.label.shape[0] == a.shape[0]
            slot_of[k] = (out_slot, den_slot)
            terms.append(_term(s, a, bb, None, out_slot, den_slot))
        slots = torch.zeros(nslots + 2 * m, device=dev, dtype=torch.float64)
        table = _device_table(terms, dev)
        _lib.check(_lib.load().mg_loss_reduce(table.data_ptr(), len(terms), slots.data_ptr(), ops._stream()), "mg_loss_reduce")
        ctx.spec, ctx.dense, ctx.keep, ctx.nslots, ctx.slot_of, ctx.inv = spec, dense, keep, nslots, slot_of, None
        ctx.shapes = [(t.shape, t.stride(), d.stride()) for t, d in zip(tensors, dense)]
        if not m:
            return slots.float()
        # loss.py:111, 114, 117, 160: each masked term divided by its own sum(label1) * c + 1e-5, on the device
        val, ctx.inv = _fold_masked(slots[nslots:nslots + m], slots[nslots + m:])
        out = slots[:nslots].clone()
        out[spec[masked[0]].slot] += val
        return out.float()

    @staticmethod
    def backward(ctx, gslots):
        dense = ctx.dense
        dev = dense[0].device
        # one flat buffer for every gradient; a tensor that appears in several terms (never the case for these losses)
        # would need accumulation - guarded below
        offs, total = [], 0
        for d in dense:
            offs.append(total)
            total += d.numel()
        flat = torch.empty(total, device=dev, dtype=torch.float32)
        seen = set()
        terms = []
        for k, (s, kb) in enumerate(zip(ctx.spec, _iter_keep(ctx.spec, ctx.keep))):
            if s.ai in seen:
                raise RuntimeError("a tensor may appear in one loss term only")
            seen.add(s.ai)
            terms.append(_term(s, dense[s.ai], kb, flat.data_ptr() + 4 * offs[s.ai], *ctx.slot_of[k]))
        table = _device_table(terms, dev)
        g = gslots.contiguous().float()
        if ctx.inv is not None:
            m = ctx.inv.numel()
            slot = next(s.slot for s in ctx.spec if s.op in MASKED_OPS)
            g = torch.cat([g, _masked_gslots(g[slot], ctx.inv), torch.zeros(m, device=dev, dtype=torch.float32)])
        _lib.check(_lib.load().mg_loss_reduce_bwd(table.data_ptr(), len(terms), g.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
        grads = []
        for i, (shape, stride, dstride) in enumerate(ctx.shapes):
            if i not in seen:
                grads.append(None)
                continue
            grads.append(torch.as_strided(flat, shape, dstride, offs[i]))
        return (None, None) + tuple(grads)


def _iter_keep(spec, keep):
    it = iter(keep)
    for s in spec:
        yield next(it) if s.b is not None else None


GAN_MODES = ("ls", "original", "w", "hinge")


class GANLoss(nn.Module):
    """loss.py:19-140 for every gan_mode: 'original' BCE with logits and 'ls' MSE against target_real_label /
    target_fake_label, 'w' -+mean, 'hinge' with the wide-edge weight map (wide_edge > 1) or, under --remove_background, the
    hair-masked terms over sum(label1) * c + 1e-5.  The mean of each scale, averaged over the discriminators."""

    def __init__(self, gan_mode, target_real_label=1.0, target_fake_label=0.0, tensor=torch.FloatTensor, opt=None):
        super().__init__()
        if gan_mode not in GAN_MODES:
            raise ValueError("Unexpected gan_mode {}".format(gan_mode))
        self.gan_mode = gan_mode
        self.real_label = target_real_label
        self.fake_label = target_fake_label
        self.opt = opt
        self._wcache = {}

    def get_weight_mask(self, input, mask):
        """loss.py:68-78: edges*wide_edge + (1-edges) at the logits' resolution, [N,h,w] (cached per label / size)."""
        n, _, h, w = input.shape
        m = mask.detach()
        key = (m.data_ptr(), m._version, tuple(m.shape), h, w)
        hit = self._wcache.get(key)
        if hit is not None:
            return hit
        m3 = m.reshape(m.shape[0], m.shape[-2], m.shape[-1]).contiguous().float()
        out = torch.empty((n, h, w), device=input.device, dtype=torch.float32)
        _lib.check(_lib.load().mg_edge_weight(m3.data_ptr(), out.data_ptr(), n, m3.shape[1], m3.shape[2], h, w,
                                              float(self.opt.wide_edge), ops._stream()), "mg_edge_weight")
        if len(self._wcache) > 8:
            self._wcache.clear()
        self._wcache[key] = out
        return out

    def _term(self, i, x, num, target_is_real, for_discriminator, label):
        """The _Spec of one scale's loss (loss.py:80-124) over num discriminators."""
        inv = 1.0 / (x.numel() * num)
        if self.gan_mode in ("original", "ls"):
            target = self.real_label if target_is_real else self.fake_label
            return _Spec(OP_BCE if self.gan_mode == "original" else OP_SQ_T, i, None, inv, 1.0, 0, target=target)
        if self.gan_mode == "w":
            return _Spec(OP_SUM, i, None, -inv if target_is_real else inv, 1.0, 0)
        if getattr(self.opt, "remove_background", False):
            lab = _hair_label(label, x)
            if for_discriminator:
                return _Spec(OP_HINGE_MASK, i, None, -1.0 / num, 1.0 if target_is_real else -1.0, 0, label=lab)
            assert target_is_real, "The generator's hinge loss must be aiming for real"
            return _Spec(OP_WSUM, i, None, -1.0 / num, 1.0, 0, label=lab)
        if for_discriminator:
            wmap = self.get_weight_mask(x, label) if self.opt.wide_edge > 1.0 else None
            return _Spec(OP_HINGE_D, i, wmap, -1.0 / (x.numel() * num), 1.0 if target_is_real else -1.0, 0)
        assert target_is_real, "The generator's hinge loss must be aiming for real"
        return _Spec(OP_SUM, i, None, -1.0 / (x.numel() * num), 1.0, 0)

    def __call__(self, input, target_is_real, for_discriminator=True, label=None):
        """loss.py:126-140: list over discriminators (each possibly a list of features, the logits last) -> mean over
        discriminators of the per-scale loss, a [1] tensor."""
        preds = input if isinstance(input, list) else [input]
        logits = [(p[-1] if isinstance(p, list) else p) for p in preds]
        num = len(logits)
        spec = [self._term(i, x, num, target_is_real, for_discriminator, label) for i, x in enumerate(logits)]
        return _LossFn.apply(spec, 1, *logits)


class GANFeatLoss(nn.Module):
    def __init__(self, opt=None):
        super().__init__()
        self.opt = opt

    def forward(self, pred_fake, pred_real, label=None):
        """loss.py:163-175: sum over discriminators and their intermediate features of L1(fake, real.detach()) * lambda_feat / num_D;
        under --remove_background the hair-masked L1_loss_mask (loss.py:154-161), each term over its own sum(label1) * c + 1e-5."""
        num_D = len(pred_fake)
        lab = _hair_label(label, pred_fake[0][0]) if getattr(self.opt, "remove_background", False) else None
        spec, tensors = [], []
        for i in range(num_D):
            for j in range(len(pred_fake[i]) - 1):
                f, r = pred_fake[i][j], pred_real[i][j].detach()
                fd = _dense(f)
                rd = _dense(r)
                if fd.stride() != rd.stride():
                    rd = r.contiguous()
                    fd = f.contiguous()
                if lab is not None:
                    spec.append(_Spec(OP_L1_MASK, len(tensors), rd, self.opt.lambda_feat / num_D, 1.0, 0, label=lab))
                else:
                    spec.append(_Spec(OP_L1, len(tensors), rd, self.opt.lambda_feat / (num_D * f.numel()), 1.0, 0))
                tensors.append(fd)
        return _LossFn.apply(spec, 1, *tensors)


# ================================================================================================ Gabor orientation loss
def gabor_bank(device, num_kernels=32, kernel_size=17):
    """The 32 Gabor kernels the reference rebuilds on every call (gabor_fn, loss.py:214-240; sigma_x 2, sigma_y 3, lambda 4,
    psi 0, theta_k = pi*k/32), with the same float32 torch arithmetic, laid out [17*17][32] for the fused kernel."""
    import math
    r = kernel_size // 2
    y = torch.arange(-r, r + 1, device=device).view(1, -1).repeat(kernel_size, 1).float()       # varies along columns
    x = torch.arange(-r, r + 1, device=device).view(-1, 1).repeat(1, kernel_size).float()       # varies along rows
    ks = []
    for k in range(num_kernels):
        theta = torch.ones(1, device=device) * (math.pi * k / num_kernels)
        x_t = x * torch.cos(theta) + y * torch.sin(theta)
        y_t = -x * torch.sin(theta) + y * torch.cos(theta)
        ks.append(torch.exp(-.5 * (x_t ** 2 / 2.0 ** 2 + y_t ** 2 / 3.0 ** 2)) * torch.cos(2 * math.pi / 4.0 * x_t + 0.0))
    return torch.stack(ks, dim=-1).reshape(kernel_size * kernel_size, num_kernels).contiguous()


class _OrientLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, bank, label2, hair):
        n, _, h, w = img.shape
        dev = img.device
        img_c = img.detach().contiguous()
        idx = torch.empty((n, h, w), device=dev, dtype=torch.uint8)
        d1 = torch.empty((n, h, w), device=dev, dtype=torch.float32)
        d2 = torch.empty((n, h, w), device=dev, dtype=torch.float32)
        sums = torch.zeros(3, device=dev, dtype=torch.float64)
        _lib.check(_lib.load().mg_orient_loss_fwd(img_c.data_ptr(), bank.data_ptr(), label2.data_ptr(), hair.data_ptr(), idx.data_ptr(),
                                                  d1.data_ptr(), d2.data_ptr(), sums.data_ptr(), n, h, w, ops._stream()), "mg_orient_loss_fwd")
        ctx.save_for_backward(bank, idx, d1, d2, sums)
        ctx.shape = (n, h, w)
        orient = (sums[0] / (2.0 * n * h * w)).float().reshape(())
        conf = (-sums[1] / sums[2]).float().reshape(())
        return orient, conf

    @staticmethod
    def backward(ctx, g_orient, g_conf):
        bank, idx, d1, d2, sums = ctx.saved_tensors
        n, h, w = ctx.shape
        wts = torch.stack([g_orient.double() / (2.0 * n * h * w), -g_conf.double() / sums[2]]).float().contiguous()
        dimg = torch.empty((n, 3, h, w), device=idx.device, dtype=torch.float32)
        _lib.check(_lib.load().mg_orient_loss_bwd(bank.data_ptr(), idx.data_ptr(), d1.data_ptr(), d2.data_ptr(), wts.data_ptr(), dimg.data_ptr(),
                                                  n, h, w, ops._stream()), "mg_orient_loss_bwd")
        return dimg, None, None, None


# ================================================================================================ DoG orientation loss
def dog_bank(device, num_kernels=32, kernel_size=17):
    """The 32 Difference-of-Gaussians kernels the reference rebuilds on every call (DoG_fn, loss.py:245-271; sigma_h 1,
    sigma_l 2, sigma_y 2, theta_k = pi*k/32), with the same float32 torch operations (one 17x17 kernel at a time, the sigmas as
    device tensors), laid out [17*17][32] like gabor_bank."""
    import math
    r = kernel_size // 2
    y = torch.arange(-r, r + 1, device=device).view(1, -1).repeat(kernel_size, 1).float()       # varies along columns
    x = torch.arange(-r, r + 1, device=device).view(-1, 1).repeat(1, kernel_size).float()       # varies along rows
    s_h, s_l, s_y = (torch.ones(1, device=device) * v for v in (1.0, 2.0, 2.0))
    ks = []
    for k in range(num_kernels):
        theta = torch.ones(1, device=device) * (math.pi * k / num_kernels)
        x_t = x * torch.cos(theta) + y * torch.sin(theta)
        y_t = -x * torch.sin(theta) + y * torch.cos(theta)
        hi = torch.exp(-.5 * (x_t ** 2 / s_h ** 2 + y_t ** 2 / s_y ** 2)) / s_h
        lo = torch.exp(-.5 * (x_t ** 2 / s_l ** 2 + y_t ** 2 / s_y ** 2)) / s_l
        ks.append((hi - lo) / (1.0 / s_h - 1.0 / s_l))
    return torch.stack(ks, dim=-1).reshape(kernel_size * kernel_size, num_kernels).contiguous()


def _orient_sincos(device, num_kernels=32):
    """[2][32]: sin and cos of 2 * (k * pi / 32), the angle of filter k as the reference forms it from the arg-max
    (loss.py:345-348), in fp32 torch arithmetic on the device."""
    import math
    a = torch.arange(num_kernels, device=device).float() * math.pi / num_kernels
    return torch.stack([torch.sin(2 * a), torch.cos(2 * a)]).contiguous()


def _pinned_table(term, device):
    """One _Term record -> device bytes, through pinned memory and an asynchronous copy (no host synchronisation; the
    caching host allocator keeps the pinned block until the copy has run)."""
    raw = torch.frombuffer(bytearray(bytes(term)), dtype=torch.uint8)
    if device.type != "cuda":           # tests/dryrun.py runs the glue on the CPU
        return raw
    return raw.pin_memory().to(device, non_blocking=True)


class _DoGOrientLossFn(torch.autograd.Function):
    """L1OLoss with the DoG filter (loss.py:320-385) in three launches forward (response pass, mg_loss_reduce op 12) and two
    backward (mg_loss_reduce_bwd op 12 -> dL/dr, then the orientation loss's bank-generic gather).  M, the sums and the tie
    count stay on the device."""

    @staticmethod
    def forward(ctx, img, bank, sincos, label2, hair):
        n, _, h, w = img.shape
        dev = img.device
        if n * h * w >= 2 ** 31:
            raise ValueError("L1OLoss (DoG): at most 2^31 - 1 pixels per call, got %d" % (n * h * w))
        idx, rh, m = ops.dog_response(img.detach().contiguous(), bank, hair)
        slots = torch.zeros(6, device=dev, dtype=torch.float64)
        term = _dog_term(rh, label2, hair, idx, m, sincos, None)
        table = _pinned_table(term, dev)
        _lib.check(_lib.load().mg_loss_reduce(table.data_ptr(), 1, slots.data_ptr(), ops._stream()), "mg_loss_reduce")
        ctx.save_for_backward(bank, sincos, label2, hair, idx, rh, m, slots)
        ctx.keep = table
        orient = (slots[0] / (2.0 * n * h * w)).float().reshape(())
        conf = (slots[1] / (slots[2] + DEN_EPS)).float().reshape(())
        return orient, conf

    @staticmethod
    def backward(ctx, g_orient, g_conf):
        bank, sincos, label2, hair, idx, rh, m, slots = ctx.saved_tensors
        n, h, w = rh.shape
        dev = rh.device
        go = g_orient.double().reshape(()) / (2.0 * n * h * w)
        gc = g_conf.double().reshape(()) / (slots[2] + DEN_EPS)
        # the gradient through M, split evenly among the pixels that attain it (torch's rule for max())
        share = (go * slots[3] + gc * slots[4]) / slots[5]
        gslots = torch.stack([go, gc, share]).float().contiguous()
        dr = torch.empty((n, h, w), device=dev, dtype=torch.float32)
        table = _pinned_table(_dog_term(rh, label2, hair, idx, m, sincos, dr.data_ptr()), dev)
        _lib.check(_lib.load().mg_loss_reduce_bwd(table.data_ptr(), 1, gslots.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
        wts = torch.cat([torch.ones(1, device=dev), torch.zeros(1, device=dev)])     # the gather's weights: dr alone
        dimg = torch.empty((n, 3, h, w), device=dev, dtype=torch.float32)
        _lib.check(_lib.load().mg_orient_loss_bwd(bank.data_ptr(), idx.data_ptr(), dr.data_ptr(), dr.data_ptr(), wts.data_ptr(),
                                                  dimg.data_ptr(), n, h, w, ops._stream()), "mg_orient_loss_bwd")
        return dimg, None, None, None, None


def _dog_term(rh, label2, hair, idx, m, sincos, ga):
    """The op 12 record: a = rh, b = label2 [N,2,H,W], label = hair [N,H,W], idx, maxv = M, table = the (sin, cos) table."""
    n, h, w = rh.shape
    t = _Term(rh.data_ptr(), label2.data_ptr(), ga, n * h * w, 1.0, 1.0, OP_ORIENT_DOG, 0)
    t.label, t.label_ns, t.h, t.w, t.H, t.W = hair.data_ptr(), h * w, h, w, h, w
    t.table, t.idx, t.maxv = sincos.data_ptr(), idx.data_ptr(), m.data_ptr()
    return t


VGG_WEIGHTS = [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]


def style_min_size_error(h, w):
    """The style loss's unbiased variance needs at least 2 pixels at relu5_1 (h/16 x w/16); the reference returns NaN below.
    The masked style loss of --remove_background has no such limit (its variance is biased)."""
    if (h // 16) * (w // 16) < 2:
        return NotImplementedError("michigan_b200: the style loss needs at least 2 pixels at relu5_1 (crop_size >= 32), got %dx%d"
                                   % (h, w))
    return None


class _VGGObjectiveFn(torch.autograd.Function):
    """Every VGG19 term of the generator objective from ONE VGG19 forward over fake || tag (|| style image) and ONE backward:

      l1       VGGLoss: sum_i w_i * mean |fake_i - tag_i|               mg_loss_reduce op 2, slot 0
      content  StyleContentLoss's loss_c: mean (fake_5 - tag_5)^2       mg_loss_reduce op 3, slot 1 (same launch)
      style    StyleContentLoss's loss_s: sum_i MSE(mu_i) + MSE(sigma_i) of fake against the style image, one mg_in_stats per tap
               over the whole batch, then one mg_style_loss_fwd launch for the five taps

    want = (l1, content, style); a term not asked for returns None.  style_img None: the style targets are the tag half (2N
    batch).  Backward: mg_loss_reduce_bwd writes the L1 tap gradients, mg_style_tap_grad adds the style gradient (and at relu5_1
    the content gradient) in place, then the hand-written VGG19 backward takes them down to d fake.

    labels = (tag label, style label), [N,1,H,W] hair labels (_hair_label): --remove_background, _MaskedVGGTerms."""

    @staticmethod
    def forward(ctx, vgg, weights, want, fake, tag, style_img, labels=None):
        l1, content, style = want
        n = fake.shape[0]
        parts = [fake.detach(), tag.detach()] + ([style_img.detach()] if style and style_img is not None else [])
        x8 = ops.nchw_to_nhwc(torch.cat(parts, 0).contiguous(), 4)
        taps, S = vgg.run(x8, n_save=n if ctx.needs_input_grad[3] else 0)
        del x8
        pairs = [(t[:n], t[n:2 * n]) for t in taps]
        ctx.masked = None
        if labels is not None:
            ctx.masked = _MaskedVGGTerms(taps, n, n if style_img is None else 2 * n, weights, want, labels)
            ctx.vgg, ctx.want, ctx.pairs, ctx.S, ctx.hw = vgg, want, pairs, S, tuple(fake.shape[2:])
            return ctx.masked.outputs
        out_l1 = out_c = out_s = None
        if l1 or content:
            terms = [_Term(a.data_ptr(), b.data_ptr(), None, a.numel(), float(w / a.numel()), 1.0, OP_L1, 0)
                     for (a, b), w in zip(pairs, weights)] if l1 else []
            if content:
                a, b = pairs[4]
                terms.append(_Term(a.data_ptr(), b.data_ptr(), None, a.numel(), 1.0 / a.numel(), 1.0, OP_SQ, 1))
            slots = torch.zeros(2 if content else 1, device=fake.device, dtype=torch.float64)
            _lib.check(_lib.load().mg_loss_reduce(_device_table(terms, fake.device).data_ptr(), len(terms), slots.data_ptr(),
                                                  ops._stream()), "mg_loss_reduce")
            if content:
                vals = slots.float()
                out_l1, out_c = (vals[0] if l1 else None), vals[1]
            else:
                out_l1 = slots.float().reshape(())
        coefs = None
        if style:
            t0 = n if style_img is None else 2 * n
            sums = [ops.channel_sums(t) for t in taps]
            loss, coefs = ops.style_loss_fwd([(s[:n], s[t0:t0 + n], t.shape[1] * t.shape[2]) for s, t in zip(sums, taps)])
            out_s = loss.float().reshape(())
        ctx.vgg, ctx.weights, ctx.want, ctx.pairs, ctx.coefs, ctx.S, ctx.hw = vgg, weights, want, pairs, coefs, S, tuple(fake.shape[2:])
        return out_l1, out_c, out_s

    @staticmethod
    def backward(ctx, g_l1, g_c, g_s):
        l1, content, style = ctx.want
        pairs = ctx.pairs
        dev = pairs[0][0].device
        grads = [None] * len(pairs)
        if ctx.masked is not None:
            grads = ctx.masked.backward(pairs, g_l1, g_c, g_s)
            ctx.pairs = ctx.masked = None
            dimg = ctx.vgg.backward(ctx.S, grads, ctx.hw)
            ctx.S = None
            return None, None, None, dimg, None, None, None
        if l1:
            grads = [torch.empty_like(a) for a, _ in pairs]
            terms = [_Term(a.data_ptr(), b.data_ptr(), ga.data_ptr(), a.numel(), float(w / a.numel()), 1.0, OP_L1, 0)
                     for (a, b), ga, w in zip(pairs, grads, ctx.weights)]
            gs = g_l1.reshape(1).contiguous().float()
            _lib.check(_lib.load().mg_loss_reduce_bwd(_device_table(terms, dev).data_ptr(), len(terms), gs.data_ptr(), ops._stream()),
                       "mg_loss_reduce_bwd")
        if content or style:
            zero = torch.zeros((), device=dev, dtype=torch.float32)
            g2 = torch.stack([g_s if style else zero, g_c if content else zero]).float().contiguous()
            for i, (a, b) in enumerate(pairs):
                coef = ctx.coefs[i] if style else None
                ct = b if content and i == len(pairs) - 1 else None
                if coef is None and ct is None:
                    continue
                grads[i] = ops.style_tap_grad(a, g2, coef=coef, content_t=ct, add=grads[i], out=grads[i])
        ctx.pairs = ctx.coefs = None
        dimg = ctx.vgg.backward(ctx.S, grads, ctx.hw)
        ctx.S = None
        return None, None, None, dimg, None, None, None


def _nchw(t):
    """The [N,C,h,w] channels-last view of an NHWC VGG tap (what the masked ops' records describe)."""
    return t.permute(0, 3, 1, 2)


class _MaskedVGGTerms:
    """The --remove_background VGG terms of one _VGGObjectiveFn call (loss.py:187-207, 634-711), l the tag label and ls the
    style label resized (nearest) to each tap:

      l1       VGGLoss.L1_loss_mask: sum_i w_i sum |x_i l - y_i l| / (sum l c + 1e-5)      op 8, one term per tap
      content  calc_content_loss: sum (x_5 l - t_5 l)^2 / (sum l c + 1e-5)                 op 9 at relu5_1
      style    calc_style_loss with calc_mean_std_mask: the fake taps' moments under ls, the style targets' under l  op 10, two
               terms per tap (the reference crosses the masks: calc_style_loss(fake, style, style_label, content_label) masks
               the fake features with the style image's hair and the style features with the tag's), then mg_style_loss_fwd
               in its masked mode

    Forward: ONE mg_loss_reduce launch for every term above (one fp64 slot buffer; the denominators folded on the device by
    _fold_masked) and one mg_style_loss_fwd.  Backward: op 8 writes the L1 tap gradients, op 10 adds the style gradients, op 9
    adds the content gradient at relu5_1: three mg_loss_reduce_bwd launches, as no two terms of one launch may write one tensor."""

    def __init__(self, taps, n, t0, weights, want, labels):
        l1, content, style = want
        lab_tag, lab_style = labels
        dev = taps[0].device
        self.want, self.weights, self.labels = want, weights, labels
        specs = []                                          # (spec, a, b, out_slot, den_slot)
        off = 0
        if l1:
            self.l1_off = off
            k = len(taps)
            for i, (t, w) in enumerate(zip(taps, weights)):
                specs.append((_Spec(OP_L1_MASK, 0, None, float(w), 1.0, 0, label=lab_tag), t[:n], t[n:2 * n], off + i, off + k + i))
            off += 2 * k
        if content:
            self.c_off = off
            t = taps[-1]
            specs.append((_Spec(OP_SQ_MASK, 0, None, 1.0, 1.0, 0, label=lab_tag), t[:n], t[n:2 * n], off, off + 1))
            off += 2
        moments = []
        if style:
            for t in taps:
                c = t.shape[3]
                for half, lab in ((t[:n], lab_style), (t[t0:t0 + n], lab_tag)):
                    specs.append((_Spec(OP_MOMENTS, 0, None, 1.0, 1.0, 0, label=lab), half, None, off, off + 2 * n * c))
                    moments.append((off, c))
                    off += 2 * n * c + n
        slots = torch.zeros(off, device=dev, dtype=torch.float64)
        terms = [_term(sp, _nchw(a), b, None, o, d) for sp, a, b, o, d in specs]
        _lib.check(_lib.load().mg_loss_reduce(_device_table(terms, dev).data_ptr(), len(terms), slots.data_ptr(), ops._stream()),
                   "mg_loss_reduce")
        out_l1 = out_c = out_s = None
        if l1:
            k = len(taps)
            val, self.inv_l1 = _fold_masked(slots[self.l1_off:self.l1_off + k], slots[self.l1_off + k:self.l1_off + 2 * k])
            out_l1 = val.float()
        if content:
            val, self.inv_c = _fold_masked(slots[self.c_off:self.c_off + 1], slots[self.c_off + 1:self.c_off + 2])
            out_c = val.float()
        self.coefs = None
        if style:
            recs = []
            for t, (fo, c), (to, _) in zip(taps, moments[0::2], moments[1::2]):
                recs.append((slots[fo:fo + 2 * n * c].view(n, 2, c), slots[to:to + 2 * n * c].view(n, 2, c), t.shape[1] * t.shape[2],
                             slots[fo + 2 * n * c:fo + 2 * n * c + n], slots[to + 2 * n * c:to + 2 * n * c + n]))
            loss, self.coefs = ops.style_loss_fwd(recs)
            out_s = loss.float().reshape(())
        self.outputs = (out_l1, out_c, out_s)

    def backward(self, pairs, g_l1, g_c, g_s):
        l1, content, style = self.want
        lab_tag, lab_style = self.labels
        dev = pairs[0][0].device
        lib = _lib.load()
        grads = [None] * len(pairs)
        if l1:
            grads = [torch.empty_like(a) for a, _ in pairs]
            gs = _masked_gslots(g_l1.reshape(()), self.inv_l1).contiguous()
            terms = [_term(_Spec(OP_L1_MASK, 0, None, float(w), 1.0, 0, label=lab_tag), _nchw(a), b, ga.data_ptr(), i, 0)
                     for i, ((a, b), ga, w) in enumerate(zip(pairs, grads, self.weights))]
            _lib.check(lib.mg_loss_reduce_bwd(_device_table(terms, dev).data_ptr(), len(terms), gs.data_ptr(), ops._stream()),
                       "mg_loss_reduce_bwd")
        if style:
            gs = g_s.reshape(1).contiguous().float()
            terms = []
            for i, (a, _) in enumerate(pairs):
                add = grads[i].data_ptr() if grads[i] is not None else None
                if grads[i] is None:
                    grads[i] = torch.empty_like(a)
                terms.append(_term(_Spec(OP_MOMENTS, 0, None, 1.0, 1.0, 0, label=lab_style), _nchw(a), self.coefs[i],
                                   grads[i].data_ptr(), 0, 0, add=add))
            _lib.check(lib.mg_loss_reduce_bwd(_device_table(terms, dev).data_ptr(), len(terms), gs.data_ptr(), ops._stream()),
                       "mg_loss_reduce_bwd")
        if content:
            a, b = pairs[-1]
            gs = _masked_gslots(g_c.reshape(()), self.inv_c).contiguous()
            add = grads[-1].data_ptr() if grads[-1] is not None else None
            if grads[-1] is None:
                grads[-1] = torch.empty_like(a)
            terms = [_term(_Spec(OP_SQ_MASK, 0, None, 1.0, 1.0, 0, label=lab_tag), _nchw(a), b, grads[-1].data_ptr(), 0, 0, add=add)]
            _lib.check(lib.mg_loss_reduce_bwd(_device_table(terms, dev).data_ptr(), 1, gs.data_ptr(), ops._stream()),
                       "mg_loss_reduce_bwd")
        self.coefs = None
        return grads


def _same_image(a, b):
    return a is b or (a.shape == b.shape and bool(torch.equal(a, b)))


def vgg_objective(vgg, fake, tag, style_image=None, l1=False, content=False, style=False, weights=VGG_WEIGHTS, label=None,
                  style_label=None):
    """(l1, content, style) of fake against tag (and the style image) from one VGG19 pass (_VGGObjectiveFn); None for a term not
    asked for.  A style image equal to the tag (paired training loads the same file for both) is not run through VGG19 again:
    the style targets then come from the tag half.

    label (the tag's [N,1,H,W] hair label) selects --remove_background: every term is masked by it, except that the fake's
    style statistics are masked by style_label (the style image's hair label), as the reference does."""
    masked = label is not None
    labels = None
    if masked:
        if style and style_label is None:
            raise ValueError("--remove_background: the style loss needs the style image's hair label")
        labels = (_hair_label(label, fake), _hair_label(style_label, fake) if style else None)
    if style and not masked:
        err = style_min_size_error(*fake.shape[2:])
        if err is not None:
            raise err
    if style:
        if style_image is None or _same_image(style_image, tag):
            style_image = None
        else:
            if style_image.shape != fake.shape:
                raise ValueError("StyleContentLoss: fake %s and style image %s differ in shape" % (tuple(fake.shape), tuple(style_image.shape)))
            style_image = style_image.float()
    if fake.shape != tag.shape:
        raise ValueError("VGG loss: fake %s and target %s differ in shape" % (tuple(fake.shape), tuple(tag.shape)))
    dev = fake.device
    if next(vgg.parameters()).device != dev:
        vgg.to(dev)
    return _VGGObjectiveFn.apply(vgg, weights, (bool(l1), bool(content), bool(style)), fake, tag.float(), style_image, labels)


def masked_vgg_losses(opt, who):
    """Whether the VGG, content and style losses run hair-masked: opt.remove_background together with opt.mask_vgg_losses.
    --remove_background alone is refused here with NotImplementedError, as before the masked terms existed, so that a
    configuration that used to be rejected does not start training a different objective unannounced; mask_vgg_losses opts
    into the reference's masked terms (install() sets it for the reference's own Pix2PixModel, whose --remove_background
    always meant them)."""
    if not getattr(opt, "remove_background", False):
        return False
    if not getattr(opt, "mask_vgg_losses", False):
        raise NotImplementedError("michigan_b200: %s with --remove_background computes the hair-masked terms only when "
                                  "opt.mask_vgg_losses is set (install() sets it for the reference's model)" % who)
    return True


class VGGLoss(nn.Module):
    """loss.py:178-207: sum_i w_i * L1(vgg(x)_i, vgg(y)_i.detach()), w = 1/32, 1/16, 1/8, 1/4, 1; under --remove_background
    (with opt.mask_vgg_losses, masked_vgg_losses) the hair-masked L1_loss_mask of each tap, sum |x_i l - y_i l| / (sum l * c
    + 1e-5), l = label resized (nearest) to the tap.  The image is fed to VGG19 in [-1, 1] without ImageNet normalisation, as
    the reference does.  The weights are never downloaded (VGG19: `state_dict` or torchvision's cache file)."""

    def __init__(self, opt=None, state_dict=None):
        super().__init__()
        self.masked = masked_vgg_losses(opt, "VGGLoss")
        from .architecture import VGG19
        self.vgg = VGG19(state_dict=state_dict)
        self.weights = list(VGG_WEIGHTS)
        self.opt = opt

    def forward(self, x, y, label=None):
        if self.masked:
            return vgg_objective(self.vgg, x, y, l1=True, weights=self.weights, label=_required(label, "VGGLoss"))[0]
        return vgg_objective(self.vgg, x, y, l1=True, weights=self.weights)[0]


def _required(label, who):
    if label is None:
        raise ValueError("%s: --remove_background needs the hair label" % who)
    return label


class StyleContentLoss(nn.Module):
    """loss.py:656-711: (loss_c, loss_s) = forward(fake_image, style_image, content_image, style_label, content_label), with
    loss_c = MSE(relu5_1(fake), relu5_1(content).detach()) and loss_s = sum over the five taps of MSE(mu_fake, mu_style) +
    MSE(sigma_fake, sigma_style) (calc_mean_std: per (n, c), unbiased variance + 1e-5).  Under --remove_background (with
    opt.mask_vgg_losses, masked_vgg_losses) the content
    term is masked by content_label over sum(label) * c + 1e-5, and the statistics are calc_mean_std_mask's (biased variance,
    the fake masked by style_label, the style image by content_label: the reference's crossing).  One VGG19 pass over fake ||
    content (|| style, unless it equals content) and one backward (_VGGObjectiveFn).  `vgg` shares another loss's VGG19."""

    def __init__(self, opt=None, vgg=None, state_dict=None):
        super().__init__()
        self.masked = masked_vgg_losses(opt, "StyleContentLoss")
        if vgg is None:
            from .architecture import VGG19
            vgg = VGG19(state_dict=state_dict)
        self.vgg = vgg
        self.opt = opt

    def forward(self, fake_image, style_image, content_image, style_label=None, content_label=None):
        if self.masked:
            _, loss_c, loss_s = vgg_objective(self.vgg, fake_image, content_image, style_image, content=True, style=True,
                                              label=_required(content_label, "StyleContentLoss"),
                                              style_label=_required(style_label, "StyleContentLoss"))
        else:
            _, loss_c, loss_s = vgg_objective(self.vgg, fake_image, content_image, style_image, content=True, style=True)
        return loss_c, loss_s


class KLDLoss(nn.Module):
    """loss.py:211-213: -0.5 sum(1 + logvar - mu^2 - e^logvar), summed over the batch and z, not averaged.  One mg_loss_reduce
    launch each way with two terms into one slot: 0.5 sum mu^2 (op 3 against zeros) and 0.5 sum (e^logvar - logvar - 1)
    (op 13), accumulated in fp64.  Under data parallelism each rank sums its own shard, as each DataParallel replica of the
    reference did before the trainer's mean()."""

    def forward(self, mu, logvar):
        if mu.shape != logvar.shape:
            raise ValueError("KLDLoss: mu %s and logvar %s differ in shape" % (tuple(mu.shape), tuple(logvar.shape)))
        zeros = torch.zeros(mu.shape, device=mu.device, dtype=torch.float32)
        spec = [_Spec(OP_SQ, 0, zeros, 0.5, 1.0, 0), _Spec(OP_KLD_EXP, 1, None, 0.5, 1.0, 0)]
        return _LossFn.apply(spec, 1, mu.float(), logvar.float())[0]


class _PixelL1Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fake, tag, mask):
        f, t = fake.detach().contiguous(), tag.detach().contiguous()
        m = mask.detach().contiguous() if mask is not None else None
        sums = ops.pixel_l1_fwd(f, t, m)
        ctx.save_for_backward(f, t, m)
        ctx.count = f.numel()
        return (sums / ctx.count).float().reshape(())

    @staticmethod
    def backward(ctx, g):
        f, t, m = ctx.saved_tensors
        gscale = (g.float() / ctx.count).reshape(1).contiguous()     # mean's backward: the fp32 gradient over the element count
        return ops.pixel_l1_bwd(f, t, gscale, m), None, None


class RGBBackgroundL1Loss(nn.Module):
    """loss.py:388-400: L1(fake * m, image_tag.detach() * m), m = input_semantics[:, 0] (the background channel of the one-hot
    label), one kernel each way (mg_pixel_l1_fwd / _bwd)."""

    def forward(self, fake, input_semantics, image_tag):
        if fake.shape != image_tag.shape or fake.shape[1] != 3:
            raise ValueError("RGBBackgroundL1Loss: expected two [N,3,H,W] images, got %s and %s" % (tuple(fake.shape), tuple(image_tag.shape)))
        return _PixelL1Fn.apply(fake, image_tag.float(), input_semantics[:, 0].float())


class RGBL1Loss(nn.Module):
    """The rgb term, nn.L1Loss()(fake, image_tag.detach()) (pix2pix_model.py:51, 328-333), on mg_pixel_l1_fwd / _bwd."""

    def forward(self, fake, image_tag):
        if fake.shape != image_tag.shape or fake.shape[1] != 3:
            raise ValueError("RGBL1Loss: expected two [N,3,H,W] images, got %s and %s" % (tuple(fake.shape), tuple(image_tag.shape)))
        return _PixelL1Fn.apply(fake, image_tag.float(), None)


LAB_WEIGHT_TH = 10.0        # train_options.py:78, the default --Lab_weight_th
_lab_weight_cache = {}


def balanced_lab(opt, who):
    """Whether `who` (LabColorLoss, HairAvgLabLoss) computes the count-balanced loss of --balance_Lab (loss.py:490-531,
    578-621): opt.balance_Lab set and opt.weight_dir naming the count table.  The reference's option parser always provides
    weight_dir (train_options.py:77), so its train.py --balance_Lab runs balanced under install().  balance_Lab without
    weight_dir is refused with NotImplementedError, as before the balanced loss existed."""
    if not getattr(opt, "balance_Lab", False):
        return False
    if getattr(opt, "weight_dir", None) is None:
        raise NotImplementedError("michigan_b200: %s with --balance_Lab needs opt.weight_dir, the [256,256] colour-count table "
                                  "(the reference's train options provide it: --weight_dir, default ./data/ab_count.npy)" % who)
    return True


def lab_weight_table(path, th=LAB_WEIGHT_TH, device="cpu"):
    """E[ka][kb] ([256,256] fp32 on `device`): the weight cal_weight (loss.py:487-513, 578-597) looks up for a pixel whose real a
    and b fall in the bins ka = int(clamp(a + 128, 0, 255)) and kb likewise.

    The count table T = np.load(path) is processed with the reference's fp32 torch operations (T == 0 -> 1, max(T) / T,
    clamped at th), then torch's own grid_sample (mode 'nearest', align_corners False, zero padding) is run once on the grid
    of all (ka, kb) bins, so E matches the reference's lookup bit for bit, including the bins its grid maps outside the
    table (bin 255 reads 0).  The reference reads the file on every forward; here it is read once per (path, th) and E is
    kept per (path, th, device)."""
    key = (os.path.realpath(path), float(th))
    dev = torch.device(device)
    hit = _lab_weight_cache.get(key + (dev,))
    if hit is not None:
        return hit
    cpu = _lab_weight_cache.get(key + (torch.device("cpu"),))
    if cpu is None:
        if not os.path.isfile(path):
            raise FileNotFoundError("--balance_Lab: colour-count table %s not found (--weight_dir)" % path)
        raw = np.load(path)
        if raw.shape != (256, 256):
            raise ValueError("--balance_Lab: the colour-count table %s must be [256,256], got %s" % (path, tuple(raw.shape)))
        w = torch.tensor(raw, dtype=torch.float32).view(1, 1, 256, 256)     # self.FloatTensor(raw)
        w[w == 0] = 1
        w = w.max() / w
        w[w > th] = th
        m = (torch.arange(256, dtype=torch.float32) - 127.5) / 127.5          # (m - 127.5) / 127.5 on the integer bins
        grid = torch.stack([m.view(1, 256).expand(256, 256), m.view(256, 1).expand(256, 256)], -1).unsqueeze(0)  # (b, a)
        cpu = F.grid_sample(w, grid, mode="nearest", padding_mode="zeros", align_corners=False)[0, 0].contiguous()
        _lab_weight_cache[key + (torch.device("cpu"),)] = cpu
    hit = cpu.to(dev)
    _lab_weight_cache[key + (dev,)] = hit
    return hit


def _lab_table_key(opt):
    return opt.weight_dir, float(getattr(opt, "Lab_weight_th", LAB_WEIGHT_TH))


class _LabLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fake, real):
        f, r = fake.detach().contiguous(), real.detach().contiguous()
        sums = ops.lab_loss_fwd(f, r)
        ctx.save_for_backward(f, r)
        ctx.count = 2 * f.shape[0] * f.shape[2] * f.shape[3]
        return (sums / ctx.count).float().reshape(())

    @staticmethod
    def backward(ctx, g):
        f, r = ctx.saved_tensors
        gscale = (g.double() / ctx.count).float().reshape(1).contiguous()
        return ops.lab_loss_bwd(f, r, gscale), None


def _balanced_lab_term(f, r, mask, table, ga):
    """The op 11 record of fake f and real r ([N,3,H,W] contiguous), mask [N,1,H,W] (rows contiguous), E on the device."""
    n, _, h, w = f.shape
    t = _Term(f.data_ptr(), r.data_ptr(), ga.data_ptr() if ga is not None else None, n * h * w, 1.0, 1.0, OP_LAB_BALANCED, 0)
    t.label, t.label_ns = mask.data_ptr(), mask.stride(0)
    t.C, t.h, t.w, t.H, t.W = 3, h, w, h, w
    t.table = table.data_ptr()
    return t


class _BalancedLabFn(torch.autograd.Function):
    """mean(w * |ab_fake - ab_real|) over N x 2 x H x W: one mg_loss_reduce launch of op 11 each way."""

    @staticmethod
    def forward(ctx, fake, real, mask, table):
        assert _lib.load().mg_loss_term_bytes() == C.sizeof(_Term)
        f, r = fake.detach().contiguous(), real.detach().contiguous()
        slots = torch.zeros(1, device=f.device, dtype=torch.float64)
        terms = _device_table([_balanced_lab_term(f, r, mask, table, None)], f.device)
        _lib.check(_lib.load().mg_loss_reduce(terms.data_ptr(), 1, slots.data_ptr(), ops._stream()), "mg_loss_reduce")
        ctx.save_for_backward(f, r, mask, table)
        ctx.count = 2 * f.shape[0] * f.shape[2] * f.shape[3]
        return (slots / ctx.count).float().reshape(())

    @staticmethod
    def backward(ctx, g):
        f, r, mask, table = ctx.saved_tensors
        ga = torch.empty_like(f)
        gslot = (g.double() / ctx.count).float().reshape(1).contiguous()
        terms = _device_table([_balanced_lab_term(f, r, mask, table, ga)], f.device)
        _lib.check(_lib.load().mg_loss_reduce_bwd(terms.data_ptr(), 1, gslot.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
        return ga, None, None, None


class LabColorLoss(nn.Module):
    """loss.py:403-531: L1 between the a, b channels of the Lab images of fake and real.detach() (xyz2lab of
    rgb2xyz((img + 1) / 2)), one fused kernel each way (csrc/mg_vgg.cu).

    With --balance_Lab and opt.weight_dir (balanced_lab) it is the count-balanced loss mean(w * |ab_fake - ab_real|), w per
    pixel = E[bins of the real pixel's a, b] * mask with 0 -> 1 (lab_weight_table; mask = the tag's hair, [N,1,H,W]), on
    mg_loss_reduce op 11 each way.  The count table is read once, at construction."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.table_key = None
        if balanced_lab(opt, "LabColorLoss"):
            self.table_key = _lab_table_key(opt)
            lab_weight_table(*self.table_key)

    def forward(self, fake, real, mask=None):
        if fake.shape != real.shape or fake.shape[1] != 3:
            raise ValueError("LabColorLoss: expected two [N,3,H,W] images, got %s and %s" % (tuple(fake.shape), tuple(real.shape)))
        if self.table_key is None:
            return _LabLossFn.apply(fake, real.float())
        n, _, h, w = fake.shape
        if mask is None or tuple(mask.shape) != (n, 1, h, w):
            raise ValueError("LabColorLoss: --balance_Lab needs the hair mask [N,1,H,W] = %s, got %s"
                             % ((n, 1, h, w), None if mask is None else tuple(mask.shape)))
        table = lab_weight_table(*self.table_key, device=fake.device)
        return _BalancedLabFn.apply(fake, real.float(), _hair_label(mask, fake), table)


class _HairAvgLabFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fake, real, mask_fake, mask_real, table):
        f, mf = fake.detach().contiguous(), mask_fake.detach().contiguous()
        sums = ops.hair_avg_lab_fwd(f, real.detach().contiguous(), mf, mask_real.detach().contiguous())
        ctx.save_for_backward(f, mf, sums)
        cnt = sums[:, :, 3:]
        avg = sums[:, :, 1:3] / torch.where(cnt == 0, torch.ones_like(cnt), cnt)       # loss.py:575
        diff = (avg[:, 0] - avg[:, 1]).abs()
        ctx.w = None
        if table is None:
            return diff.mean().float()
        # loss.py:589-597 on the real averages (fp32, as the reference holds them): N gathers, no host synchronisation
        k = (avg[:, 1].float() + 128).clamp(0, 255).int().long()
        ctx.w = table[k[:, 0], k[:, 1]]
        return (diff * ctx.w.double().unsqueeze(1)).mean().float()

    @staticmethod
    def backward(ctx, g):
        f, mf, sums = ctx.saved_tensors
        if ctx.w is None:
            return ops.hair_avg_lab_bwd(f, mf, sums, g.float().reshape(1).contiguous()), None, None, None, None
        # image n's gradient is the unbalanced one of a batch of 1 scaled by w[n] / N: one launch per image
        n = f.shape[0]
        gs = (g.double() * ctx.w.double() / n).float().contiguous()
        dfake = torch.empty_like(f)
        for i in range(n):
            ops.hair_avg_lab_bwd(f[i:i + 1], mf[i:i + 1], sums[i:i + 1], gs[i:i + 1], out=dfake[i:i + 1])
        return dfake, None, None, None, None


class HairAvgLabLoss(nn.Module):
    """loss.py:534-621: L1 between the hair-averaged a, b of fake (tag hair mask_fake) and of real.detach() (reference hair
    mask_real), avg = sum(Lab * m) / sum(m), a mask sum of 0 counted as 1.  One fused kernel pair each way (csrc/mg_vgg.cu:
    mg_hair_avg_lab_fwd, mg_hair_avg_lab_bwd).

    With --balance_Lab and opt.weight_dir (balanced_lab): mean(w[n] * |avg_ab_fake - avg_ab_real|), w[n] = E[bins of image n's
    real average a, b] (lab_weight_table; no mask factor, no 0 -> 1), gathered on the device from the forward's sums; the
    backward runs mg_hair_avg_lab_bwd once per image with the gradient scaled by w[n].  The count table is read once, at
    construction."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.table_key = None
        if balanced_lab(opt, "HairAvgLabLoss"):
            self.table_key = _lab_table_key(opt)
            lab_weight_table(*self.table_key)

    def forward(self, fake, real, mask_fake, mask_real):
        if fake.shape != real.shape or fake.shape[1] != 3:
            raise ValueError("HairAvgLabLoss: expected two [N,3,H,W] images, got %s and %s" % (tuple(fake.shape), tuple(real.shape)))
        n, _, h, w = fake.shape
        for name, m in (("mask_fake", mask_fake), ("mask_real", mask_real)):
            if tuple(m.shape) != (n, 1, h, w):
                raise ValueError("HairAvgLabLoss: %s must be [N,1,H,W] = %s, got %s" % (name, (n, 1, h, w), tuple(m.shape)))
        table = None if self.table_key is None else lab_weight_table(*self.table_key, device=fake.device)
        return _HairAvgLabFn.apply(fake, real.float(), mask_fake.float(), mask_real.float(), table)


class L1OLoss(nn.Module):
    """loss.py:274-385: (orient_loss, confidence_loss) = forward(fake_image, orientation_label, input_semantics).
    orientation_label: the 1-channel angle map (0..255) or, with --use_ig, the 2-channel (sin 2t, cos 2t) map.

    orient_filter containing 'gabor' selects the Gabor bank (confidence (tanh(r) + 1) / 2, log confidence loss); any other value
    the Difference-of-Gaussians bank, whose confidence r * hair / M is normalised by M, the maximum over the batch of this call,
    with the L1 confidence loss against the hair mask.  Under data parallelism M is taken over each rank's shard, as each of the
    reference's DataParallel replicas took it over its own; it is not reduced across ranks.  A batch without hair has M = 0 and
    both losses and the gradient are NaN, as in the reference."""

    def __init__(self, opt, channel_in=1, channel_out=1, stride=1, padding=8):
        super().__init__()
        self.opt = opt
        self.dog = "gabor" not in getattr(opt, "orient_filter", "gabor")
        self._bank = None
        self._sincos = None

    def forward(self, fake_image0, orientation_label0, input_semantics):
        import math
        dev = fake_image0.device
        if self._bank is None or self._bank.device != dev:
            self._bank = dog_bank(dev) if self.dog else gabor_bank(dev)
            self._sincos = _orient_sincos(dev) if self.dog else None
        hair = input_semantics[:, 1].contiguous().float()
        if not self.opt.use_ig:
            t = orientation_label0.float() / 255 * math.pi
            label2 = torch.cat([torch.sin(2 * t), torch.cos(2 * t)], dim=1).contiguous()
        else:
            label2 = orientation_label0.float().contiguous()
        if self.dog:
            return _DoGOrientLossFn.apply(fake_image0, self._bank, self._sincos, label2.detach(), hair.detach())
        return _OrientLossFn.apply(fake_image0, self._bank, label2.detach(), hair.detach())
