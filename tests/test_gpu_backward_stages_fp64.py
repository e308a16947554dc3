"""Every hand-written backward stage of the training path (networks/autograd.py and the encoders' backward_nhwc) against
float64 CPU autograd of the stage's forward, evaluated at the state the package's own training forward saved.

Each case runs the package's forward in save mode (SPADEBGenerator.run, MultiscaleDiscriminator.run, ConvEncoder.run, an
encoder's forward_nhwc), draws the incoming gradient from a seeded CPU generator, calls the real backward function with a
fresh _Grads, and compares every parameter gradient it leaves and every input gradient it returns.

The reference is the stage's forward in plain torch.nn.functional, differentiated in fp64 at the saved state:
  * every tensor a gradient kernel reads is the saved fp32 value (`st`: the value of the saved tensor, the gradient of the
    fp64 expression), so operand rounding of the forward never enters the comparison and errors do not compound from one
    stage to the next;
  * every ReLU / LeakyReLU derivative comes from the forward's own saved output (the SPADE h, the encoders' y, the
    discriminator's f0), or, after an InstanceNorm, from the same fp32 fma the kernels evaluate on the saved input and its
    (rstd, shift) table: the reference differentiates the piecewise function the kernels chose;
  * batch norm and instance norm in train mode (statistics in fp64 from the saved input); spectral norm as torch's
    spectral_norm, with u and v constant.

Bound: |got - ref| <= k * u * R_abs + tiny per element.  R_abs is the same fp64 computation on absolute values (|dy|, |W|,
|x|, masks as 0 / 1 or 1 / 0.2), the normalisations and spectral norm replaced by the magnitude of each term of their
adjoints (tests/test_gpu_backward_kernels.py).  It does not compound down a stack of layers: at every saved tensor the
magnitude pass restarts from the signed reference's gradient there (`st`), so each R_abs spans one layer's gradient GEMMs
and normalisation, and an early layer is held as tightly as a late one.  u is the coarsest operand rounding of the stage's
gradient GEMMs: 2^-8 where a one-pass bf16 operand enters (mixed16: dgamma|dbeta, and conv_0 / conv_1 / conv_s gradients
unless MICHIGAN_B200_GRAD16=gb), 2^-11 for TF32.  k is HEADROOM times the ratio measured on an H100 for that tensor of that
case (MEASURED, at the end; -s prints every ratio next to its k).

The mlp_shared ReLU derivative is the one the kernels chose: the mask comes from the same mlp_shared recomputation
_spade_conv_bwd runs (_actv_mask).  Every case reloads the weights and spectral-norm vectors first, so its state does not
depend on which cases ran before it.

Wall time of the module: 64 s on an H100 80GB HBM3 host (700 W power limit, 8 CPU threads), mostly the fp64 CPU
references.  The measured ratios are reproduced bit for bit from one run to the next.
"""
import random
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from michigan_b200 import networks, ops, precision
from michigan_b200.networks import autograd
from fp64ref import U_BF16, U_TF32, check_close, d64, nhwc
from helpers import preprocessed, reference_layout_state

pytestmark = pytest.mark.gpu

DEV = "cuda"
EPS = 1e-5
CFG = dict(ngf=64, ndf=64, size=128, batch=2, data_seed=9)
BLOCKS = ["head_0", "G_middle_0", "G_middle_1", "up_0", "up_1", "up_2", "up_3"]


# ============================================================================================== fp64 reference pieces
def c64(t):
    """NHWC tensor -> NCHW fp64 CPU."""
    return d64(t).permute(0, 3, 1, 2).contiguous()


_PASS = None     # the reference pass in progress (Ref)


class _Restart(torch.autograd.Function):
    """Magnitude pass at a saved tensor: the value |saved|; the adjoint |g| + (per-channel mean of |g|), g the signed
    reference's gradient at the same point, whatever magnitude arrives from below."""

    @staticmethod
    def forward(ctx, expr, saved, g):
        a = g.abs()
        dims = (0, 2, 3) if a.dim() == 4 else tuple(i for i in range(a.dim()) if i != a.dim() - 1)
        ctx.mag = a + (a.mean(dims, keepdim=True) if dims else a)
        return saved.clone()

    @staticmethod
    def backward(ctx, g):
        return ctx.mag, None, None


def st(expr, saved):
    """The value of `saved` (a tensor the forward kept and the backward reads) with the gradient of `expr`.

    In the magnitude pass (Ref) every such tensor is a restart: the magnitude below it is that of the signed reference's
    gradient there (plus its channel mean, the scale of the GEMM errors of its neighbours), not the magnitude of everything
    above.  Each R_abs therefore spans one layer's gradient GEMMs and normalisation, and does not compound down a stack:
    one k holds every layer of a case."""
    p = _PASS
    if p is not None and p.A:
        i = p.i
        p.i += 1
        g = p.rec[i] if p.rec[i] is not None else torch.zeros_like(saved)
        return _Restart.apply(expr, saved, g)
    out = expr + (saved - expr).detach()
    if p is not None and out.requires_grad:
        i = len(p.rec)
        p.rec.append(None)
        out.register_hook(lambda g, i=i, rec=p.rec: rec.__setitem__(i, g.detach()))
    elif p is not None:
        p.rec.append(None)
    return out


def up(t, s):
    """Nearest 2^s upsample of an NCHW tensor."""
    f = 1 << s
    return t.repeat_interleave(f, 2).repeat_interleave(f, 3) if s else t


def lrelu_mask(pos):
    return torch.where(pos, torch.ones((), dtype=torch.float64), torch.full((), 0.2, dtype=torch.float64))


def in_pos(y, ss):
    """Sign of the kernels' x-hat = fmaf(y, rstd, shift) for NHWC y and its [N,2,C] table, as an NCHW mask: the fp64
    product of two fp32 values is exact, so the fp64 sum has the sign of the fused multiply-add."""
    y, ss = d64(y), d64(ss)
    xh = y * ss[:, 0][:, None, None, :] + ss[:, 1][:, None, None, :]
    return (xh > 0).permute(0, 3, 1, 2)


class _NormMag(torch.autograd.Function):
    """Magnitude of a train-mode normalisation: forward xa = (|x| + |mean|) rstd, adjoint
    rstd (g + mean(g) + xa mean(g xa)), the terms of the normalisation's adjoint in absolute value."""

    @staticmethod
    def forward(ctx, xa, mean, rstd, dims):
        out = (xa + mean.abs()) * rstd
        ctx.save_for_backward(out, rstd)
        ctx.dims = dims
        return out

    @staticmethod
    def backward(ctx, g):
        xa, rstd = ctx.saved_tensors
        d = ctx.dims
        return rstd * (g + g.mean(d, keepdim=True) + xa * (g * xa).mean(d, keepdim=True)), None, None, None


def norm(x, dims, A, ref):
    """Train-mode batch norm (dims (0, 2, 3)) or instance norm (dims (2, 3)) of NCHW x without affine, eps 1e-5; under A
    the magnitude map, with the statistics of the signed tensor ref (x's value in the signed pass)."""
    if not A:
        m = x.mean(dims, keepdim=True)
        return (x - m) / torch.sqrt(x.var(dims, unbiased=False, keepdim=True) + EPS)
    m = ref.mean(dims, keepdim=True)
    rstd = 1.0 / torch.sqrt(ref.var(dims, unbiased=False, keepdim=True) + EPS)
    return _NormMag.apply(x, m, rstd, dims)


class _SNMag(torch.autograd.Function):
    """Magnitude of W / sigma, sigma = u^T W v (u, v constant): adjoint g / sigma + |u| |v|^T sum(g |W|) / sigma^2."""

    @staticmethod
    def forward(ctx, wa, sigma, ua, va):
        ctx.save_for_backward(wa, ua, va)
        ctx.sigma = sigma
        return wa / sigma

    @staticmethod
    def backward(ctx, g):
        wa, ua, va = ctx.saved_tensors
        s = ctx.sigma
        return g / s + (ua[:, None] * va[None, :]).view(g.shape) * float((g * wa).sum()) / s ** 2, None, None, None


def sn_weight(w, conv, A):
    """W / sigma of a spectral-norm conv with the u, v its forward left (torch's spectral_norm), or its magnitude."""
    u, v = d64(conv.weight_u), d64(conv.weight_v)
    if not A:
        return w / (u @ w.view(w.shape[0], -1) @ v)
    sigma = float(u @ d64(conv.weight_orig).view(w.shape[0], -1) @ v)
    return _SNMag.apply(w, sigma, u.abs(), v.abs())


class Ref:
    """fp64 autograd of fwd(P, A) over the leaves P: the signed pass (A False), which records the gradient at every `st`
    point, then the magnitude pass (A True: every leaf and every saved value in absolute value, the output gradients too,
    restarted at every `st` point from the signed pass's gradient there)."""

    def __init__(self, leaves, fwd, douts):
        global _PASS
        self.grad, self.rabs = {}, {}
        self.rec, self.A, self.i = [], False, 0
        try:
            for A, out in ((False, self.grad), (True, self.rabs)):
                self.A, self.i = A, 0
                _PASS = self
                P = {k: (d64(v).abs() if A else d64(v)).requires_grad_(True) for k, v in leaves.items()}
                outs = fwd(P, A)
                gs = torch.autograd.grad(outs, list(P.values()), [d.abs() if A else d for d in douts], allow_unused=True)
                for k, g in zip(P, gs):
                    out[k] = g
            assert self.i == len(self.rec), (self.i, len(self.rec))    # both passes met the same st points
        finally:
            _PASS = None


def value(A):
    """Saved tensor -> its fp64 value in the pass (NCHW for 4-d NHWC tensors when nchw=True)."""
    def V(t, nchw=True):
        r = c64(t) if (nchw and t.dim() == 4) else d64(t)
        return r.abs() if A else r
    return V


def param_names(module):
    return {id(p): n for n, p in module.named_parameters()}


def check(tag, tensor, got, ref, rabs, u):
    """check_close with k = HEADROOM x the ratio measured for this tensor of this case (MEASURED)."""
    return check_close("%s %s" % (tag, tensor), got, ref, rabs, max(HEADROOM * MEASURED[tag][tensor], 1e-12), u)


def check_params(tag, module, G, ref, u, skip=()):
    """Every parameter gradient of `module` left in G (autograd._Grads) against the reference; parameters the stage does
    not reach (skip, by name prefix) must have none."""
    for n, p in module.named_parameters():
        got = G.get(p)
        if n.startswith(skip):
            assert got is None, (tag, n)
            continue
        assert got is not None, "%s: no gradient for %s" % (tag, n)
        check(tag, n, got.reshape(p.shape), ref.grad[n], ref.rabs[n], u)


# ============================================================================================== generator forward
_G = {}


def _generator(use_vae=False):
    from michigan_b200.options import make_opt
    if use_vae not in _G:
        opt = make_opt(is_train=True, ngf=CFG["ngf"], ndf=CFG["ndf"], crop_size=CFG["size"], batchSize=CFG["batch"], use_vae=use_vae)
        G = networks.SPADEBGenerator(opt)
        if use_vae:
            from michigan_b200.synth import fill_state_dict
            sd = {k: v.detach().clone() for k, v in G.state_dict().items()}
            fill_state_dict(sd, 41)
        else:
            sd = reference_layout_state("G", CFG, 31)
        _G[use_vae] = (G.to(DEV).train(), sd)
    G, sd = _G[use_vae]
    G.load_state_dict(sd)      # every case starts from the same weights and spectral-norm u, v, whatever ran before
    return G


def _run_generator(G, z=None):
    _, pre = preprocessed(CFG)
    p = {k: v.to(DEV) for k, v in pre.items()}
    random.seed(4)
    st_ = SimpleNamespace()
    with torch.no_grad():
        G.run(p["input_ref"], p["orient_mask"], p["image_ref"], p["input_tag"], p["noise"], p["image_tag"], st_, z=z)
    torch.cuda.synchronize()
    return st_


def _precision(mode, grad16, monkeypatch):
    old = precision.mode()
    precision.set_mode(mode)
    if grad16 is not None:
        monkeypatch.setenv("MICHIGAN_B200_GRAD16", grad16)
    else:
        monkeypatch.delenv("MICHIGAN_B200_GRAD16", raising=False)
    return old


# ============================================================================================== SPADE blocks
def _spade_ref(P, names, sp, S, x, xs, seg, A, memo, key):
    """h = act(BN(up(x)) (1 + gamma) + beta) of one SPADE (NCHW fp64), gamma, beta = mlp_gamma / mlp_beta(relu(mlp_shared(
    seg'))), seg' the nearest resize of the segmap; the values of 1 + gamma and h are the saved ones."""
    V = value(A)
    pn = lambda p: P[names[id(p)]]   # noqa: E731
    segr = V(seg)[:, :, ::S.R, ::S.R]
    pre = F.conv2d(segr, pn(sp.mlp_shared[0].weight), pn(sp.mlp_shared[0].bias), padding=1)
    actv = pre * memo[key]                 # the ReLU mask of the kernels' own recomputation of actv
    gamma = F.conv2d(actv, pn(sp.mlp_gamma.weight), pn(sp.mlp_gamma.bias), padding=1)
    beta = F.conv2d(actv, pn(sp.mlp_beta.weight), pn(sp.mlp_beta.bias), padding=1)
    g1 = st(1 + gamma, V(S.g1))
    xhat = norm(up(x, xs), (0, 2, 3), A, up(c64(S.src), xs))
    p = xhat * g1 + beta
    if S.act == ops.ACT_LRELU:
        p = p * lrelu_mask(c64(S.h) > 0)
    return st(p, V(S.h))


def _actv_mask(S, seg4):
    """actv > 0 of the mlp_shared recomputation _spade_conv_bwd hands the fused ReLU backward of the mlp_shared weight
    gradient (same call, same operand format), as an NCHW fp64 mask: the reference's ReLU derivative is the one the kernels
    chose, not one of an fp64 recomputation that could differ where the pre-activation is within rounding of 0."""
    b = S.sp.mlp_shared[0].bias.detach()
    gfmt = precision.grad_fmt()
    if gfmt == ops.TF32:
        actv = ops.mlp_shared(seg4, S.wsh, b, seg_resize=S.R, act=ops.ACT_RELU, round_out=True, out_hw=S.hw)
    else:
        actv = ops.mlp_shared(seg4, S.wsh, b, seg_resize=S.R, act=ops.ACT_RELU, out_hw=S.hw, out16=(gfmt, False))[0]
    return (c64(actv) > 0).double()


def _block_ref(blk, S, seg, masks):
    names = param_names(blk)

    def conv_w(P, conv, A):
        w = P[names[id(conv.weight_orig)]]
        return sn_weight(w, conv, A)

    def fwd(P, A):
        V = value(A)
        memo = fwd.memo
        x = P["x"]
        h0 = _spade_ref(P, names, blk.norm_0, S.sp0, x, S.xs, seg, A, memo, "0")
        c0 = F.conv2d(h0, conv_w(P, blk.conv_0, A), P[names[id(blk.conv_0.bias)]], padding=1)
        dx = st(c0, V(S.dx))
        h1 = _spade_ref(P, names, blk.norm_1, S.sp1, dx, 0, seg, A, memo, "1")
        y = F.conv2d(h1, conv_w(P, blk.conv_1, A), P[names[id(blk.conv_1.bias)]], padding=1)
        if blk.learned_shortcut:
            hs = _spade_ref(P, names, blk.norm_s, S.sps, x, S.xs, seg, A, memo, "s")
            y = y + F.conv2d(hs, conv_w(P, blk.conv_s, A))
        else:
            y = y + up(x, S.xs)
        if S.blend is not None:
            _, hair, back, ms = S.blend
            hs_ = d64(hair)[:, None, ::ms, ::ms]
            bs_ = d64(back)[:, None, ::ms, ::ms]
            y = P["bf"] * (1 - hs_) + y * (1 - bs_)
        return [y]
    fwd.memo = masks
    leaves = {n: p for n, p in blk.named_parameters()}
    leaves["x"] = c64(S.x)
    if S.blend is not None:
        leaves["bf"] = c64(S.blend[0])
    return leaves, fwd


# mode, MICHIGAN_B200_GRAD16, blocks, u
_MODES = {
    "mixed16": ("mixed16", None, BLOCKS, U_BF16),
    "tf32": ("tf32", None, ["G_middle_0", "up_1"], U_TF32),
    "mixed16_grad16_gb": ("mixed16", "gb", ["head_0", "up_0"], U_BF16),
}
_BLOCK_CASES = [(m, b) for m, (_, _, bs, _) in _MODES.items() for b in bs]


@pytest.mark.parametrize("mode,block", _BLOCK_CASES, ids=["%s-%s" % c for c in _BLOCK_CASES])
def test_spade_block_bwd(mode, block, monkeypatch):
    """block_bwd (blend_bwd, _spade_conv_bwd of conv_1 / conv_0 / conv_s with spade_bwd and the gamma|beta and mlp_shared
    gradient GEMMs, bn_bwd_apply of both batch norms and of the identity shortcut): dx, dbf and every parameter gradient
    of one generator block.  head_0 reads its input at x_shift 0, the others at 1; up_0 .. up_3 have a learned shortcut and
    the background blend, the first three the identity shortcut.  mixed16 covers one-pass fp16 (up_1 .. up_3) and three-pass
    bf16 (head_0 .. up_0) forwards with bf16 gradient GEMMs; tf32 the TF32 branch of _spade_conv_bwd; GRAD16=gb TF32 conv
    gradients under mixed16."""
    pmode, g16, _, u = _MODES[mode]
    old = _precision(pmode, g16, monkeypatch)
    try:
        G = _generator()
        st_ = _run_generator(G)
        idx = BLOCKS.index(block)
        blk, S = getattr(G, block), st_.saved[idx]
        if pmode == "mixed16" and g16 is None and blk.conv_0.weight_orig.shape[1] % 64 == 0:
            assert getattr(S.sp0, "h16", None) is not None        # the bf16 weight-gradient operand is reused
        gen = torch.Generator().manual_seed(100 + idx)
        N, h, w = S.x.shape[0], S.hw[0], S.hw[1]
        dout = torch.randn(N, h, w, blk.fout, generator=gen)
        grads = autograd._Grads()
        dx, dbf = autograd.block_bwd(grads, blk, S, dout.to(DEV), st_.seg4, st_.inv_of)
        masks = {key: _actv_mask(Sp, st_.seg4) for key, Sp in (("0", S.sp0), ("1", S.sp1), ("s", getattr(S, "sps", None)))
                 if Sp is not None}
        torch.cuda.synchronize()
    finally:
        precision.set_mode(old)
    leaves, fwd = _block_ref(blk, S, st_.seg4, masks)
    ref = Ref(leaves, fwd, [c64(dout)])
    tag = "%s %s" % (mode, block)
    check(tag, "dx", dx, nhwc(ref.grad["x"]), nhwc(ref.rabs["x"]), u)
    if S.blend is not None:
        check(tag, "dbf", dbf, nhwc(ref.grad["bf"]), nhwc(ref.rabs["bf"]), u)
    else:
        assert dbf is None
    check_params(tag, blk, grads, ref, u)


# ============================================================================================== encoders


def test_image_encoder3_fc_bwd():
    """fc_bwd (ImageEncoder3, --Image_encoder_mode partialconv): the bilinear resize of the 4x4 map to the 2x2 latent, the
    masked mean, the last InstanceNorm, then per partial conv (acc * ratio + b) * upd with the masks the forward saved,
    InstanceNorm + LeakyReLU times the previous update mask, and the thin conv of layer1.  TF32 gradient GEMMs."""
    G = _generator()
    st_ = _run_generator(G)
    E, S = G.fc, st_.Sfc
    assert isinstance(E, networks.ImageEncoder3)
    gen = torch.Generator().manual_seed(7)
    out_shape = (CFG["batch"], G.sh, G.sw, E.layer5.out_channels)
    assert (G.sh, G.sw) != S.mhw                                       # the resize backward is reached
    dout = torch.randn(out_shape, generator=gen)
    grads = autograd._Grads()
    E.backward_nhwc(grads, S, dout.to(DEV))
    torch.cuda.synchronize()
    names = param_names(E)

    def fwd(P, A):
        V = value(A)
        pw = lambda p: P[names[id(p)]]                                 # noqa: E731
        mr = d64(S.mref)
        y = F.conv2d(V(S.x0)[:, :3], pw(E.layer1.weight), None, stride=2, padding=1)
        y = (y * d64(S.l1.ratio)[:, None] + pw(E.layer1.bias)[None, :, None, None]) * d64(S.l1.upd)[:, None]
        for L in S.layers:
            a = norm(y, (2, 3), A, c64(L.y_in)) * lrelu_mask(in_pos(L.y_in, L.ss)) * d64(L.pm_in)[:, None]
            a = st(a, V(L.a))
            y = F.conv2d(a, pw(L.layer.weight), None, stride=2, padding=1)
            y = (y * d64(L.ratio)[:, None] + pw(L.layer.bias)[None, :, None, None]) * d64(L.upd)[:, None]
        a6 = norm(y, (2, 3), A, c64(S.y5)) * lrelu_mask(in_pos(S.y5, S.ss6))
        h = a6.shape[2]
        rr = mr.shape[1] // h
        mref = mr[:, None, ::rr, ::rr]
        mtag = d64(S.mtag)[:, None, ::rr, ::rr]
        out = (a6 * mref).sum((2, 3), keepdim=True) / mref.sum((2, 3), keepdim=True).clamp_min(1.0) * mtag
        return [F.interpolate(out, size=(G.sh, G.sw), mode="bilinear", align_corners=False)]
    ref = Ref({n: p for n, p in E.named_parameters()}, fwd, [d64(dout).permute(0, 3, 1, 2)])
    check_params("ImageEncoder3", E, grads, ref, U_TF32)


def _stack_ref(E, S, names, P, A, n_layers):
    """SNConvStack.run_stack at the saved state: the thin conv of layer1, then lrelu(IN(y)) -> SN conv per layer; returns
    the last conv's output (NCHW fp64)."""
    V = value(A)
    convs = E.convs()[:n_layers]
    y = F.conv2d(V(S.x0)[:, :3], sn_weight(P[names[id(convs[0].weight_orig)]], convs[0], A), None, stride=2, padding=1)
    for L in S.layers:
        a = st(norm(y, (2, 3), A, c64(L.y_in)) * lrelu_mask(in_pos(L.y_in, L.ss)), V(L.a))
        y = F.conv2d(a, sn_weight(P[names[id(L.conv.weight_orig)]], L.conv, A), None, stride=2, padding=1)
    return y


def _filled(E, seed):
    from michigan_b200.synth import fill_state_dict
    sd = {k: v.detach().clone() for k, v in E.state_dict().items()}
    fill_state_dict(sd, seed)
    E.load_state_dict(sd)
    return E.to(DEV).train()


def _opt(**kw):
    from michigan_b200.options import make_opt
    return make_opt(is_train=True, ngf=64, ndf=64, **kw)


def _ref_images(N, H, seed):
    gen = torch.Generator().manual_seed(seed)
    img = torch.rand(N, 3, H, H, generator=gen) * 2 - 1
    lab_ref = torch.zeros(N, 1, H, H)
    lab_ref[:, :, H // 5:H * 3 // 5, H // 6:H * 4 // 5] = 1
    lab_ref[1] = torch.roll(lab_ref[1], H // 8, dims=-1)
    lab_tag = torch.zeros(N, 1, H, H)
    lab_tag[:, :, H // 4:H * 2 // 3, H // 5:H * 3 // 4] = 1
    return img.to(DEV), lab_ref.to(DEV), lab_tag.to(DEV), gen




@pytest.mark.parametrize("pick", [True, False], ids=["pick", "no_pick"])
def test_image_encoder2_bwd(pick):
    """ImageEncoder2.backward_nhwc (--Image_encoder_mode instance): the strided pick of the 4x4 map to a 2x2 latent (or none
    when the latent is 4x4), the masked mean, the last InstanceNorm and sn_conv_stack_bwd with spectral_norm_bwd of every
    layer.  TF32 gradient GEMMs."""
    s = 2 if pick else 4
    E = _filled(networks.ImageEncoder2(_opt(crop_size=CFG["size"], Image_encoder_mode="instance"), s, s), 51)
    img, lr, lt, gen = _ref_images(CFG["batch"], CFG["size"], 52)
    S = SimpleNamespace()
    with torch.no_grad():
        out = E.forward_nhwc(img, lr, lt, save=S)
    assert (S.pick is not None) == pick
    dout = torch.randn(out.shape, generator=gen)
    grads = autograd._Grads()
    E.backward_nhwc(grads, S, dout.to(DEV))
    torch.cuda.synchronize()
    names = param_names(E)

    def fwd(P, A):
        y = _stack_ref(E, S, names, P, A, 5)
        a = norm(y, (2, 3), A, c64(S.y_last)) * lrelu_mask(in_pos(S.y_last, S.ss_last))
        rr = S.mref.shape[1] // a.shape[2]
        mref = d64(S.mref)[:, None, ::rr, ::rr]
        mtag = d64(S.mtag)[:, None, ::rr, ::rr]
        o = (a * mref).sum((2, 3), keepdim=True) / mref.sum((2, 3), keepdim=True).clamp_min(1.0) * mtag
        if S.pick is not None:
            o = o[:, :, ::S.pick[0], ::S.pick[1]]
        return [o]
    ref = Ref({n: p for n, p in E.named_parameters()}, fwd, [d64(dout).permute(0, 3, 1, 2)])
    check_params("ImageEncoder2 pick=%s" % pick, E, grads, ref, U_TF32)


def test_image_encoder_latent_bwd():
    """ImageEncoder.backward_nhwc (--Image_encoder_mode norm): latent_bwd of the fc over the pooled rows (NCHW row order of
    the reference's view), the adjoint of the pooled mean's pixel (0, 0), the last InstanceNorm and sn_conv_stack_bwd at the
    256x256 resize of the image.  TF32 gradient GEMMs."""
    E = _filled(networks.ImageEncoder(_opt(crop_size=CFG["size"], Image_encoder_mode="norm"), 2, 2), 53)
    img, lr, lt, gen = _ref_images(CFG["batch"], CFG["size"], 54)
    S = SimpleNamespace()
    with torch.no_grad():
        out = E.forward_nhwc(img, lr, lt, save=S)
    dout = torch.randn(out.shape, generator=gen)
    grads = autograd._Grads()
    E.backward_nhwc(grads, S, dout.to(DEV))
    torch.cuda.synchronize()
    names = param_names(E)
    N = out.shape[0]

    def fwd(P, A):
        V = value(A)
        y = _stack_ref(E, S, names, P, A, 5)
        a = norm(y, (2, 3), A, c64(S.y_last)) * lrelu_mask(in_pos(S.y_last, S.ss_last))
        pooled = st(a.mean((2, 3)), V(S.z4, nchw=False).view(N, -1))
        o = F.conv2d(pooled[:, :, None, None], P["fc.weight"], P["fc.bias"])
        return [o.view(N, -1, E.sh, E.sw)]
    ref = Ref({n: p for n, p in E.named_parameters() if not n.startswith("layer6.")}, fwd, [d64(dout).permute(0, 3, 1, 2)])
    check_params("ImageEncoder", E, grads, ref, U_TF32, skip=("layer6.",))


def test_vae_latent_head_bwd(monkeypatch):
    """latent_bwd of the --use_vae head as _GeneratorFn.backward calls it: x = view(z W^T + b) in the reference's NCHW order;
    dW, db and dz.  TF32 GEMMs."""
    G = _generator(use_vae=True)
    gen = torch.Generator().manual_seed(61)
    z = torch.randn(CFG["batch"], G.opt.z_dim, generator=gen)
    st_ = _run_generator(G, z=z.to(DEV))
    S = st_.Sfc
    C = 16 * CFG["ngf"]
    dx = torch.randn(CFG["batch"], G.sh, G.sw, C, generator=gen)
    grads = autograd._Grads()
    dz = autograd.latent_bwd(grads, G.fc, S, dx.to(DEV))
    torch.cuda.synchronize()

    def fwd(P, A):
        return [(P["z"] @ P["w"].t() + P["b"]).view(-1, C, G.sh, G.sw)]
    ref = Ref({"z": S.z4.view(CFG["batch"], -1), "w": G.fc.weight, "b": G.fc.bias}, fwd, [d64(dx).permute(0, 3, 1, 2)])
    check("vae head", "dW", grads.get(G.fc.weight), ref.grad["w"], ref.rabs["w"], U_TF32)
    check("vae head", "db", grads.get(G.fc.bias), ref.grad["b"], ref.rabs["b"], U_TF32)
    check("vae head", "dz", dz, ref.grad["z"], ref.rabs["z"], U_TF32)




def test_background_encoder_bg_bwd():
    """bg_bwd: the four blend gradients (x3, x2, x1, x0) all non-zero, each added into its layer's reflect-pad backward;
    ReLU masks from the saved outputs; the 7x7 reflect-padded thin conv of conv1.  TF32 gradient GEMMs."""
    G = _generator()
    st_ = _run_generator(G)
    bg, S = G.backgroud_enc, st_.Sbg
    feats = [S.layers[2].y, S.layers[1].y, S.layers[0].y, S.x0]
    gen = torch.Generator().manual_seed(71)
    dfeats = [torch.randn(f.shape, generator=gen) for f in feats]
    grads = autograd._Grads()
    autograd.bg_bwd(grads, bg, S, [d.to(DEV) for d in dfeats])
    torch.cuda.synchronize()
    names = param_names(bg)

    def fwd(P, A):
        V = value(A)
        pw = lambda p: P[names[id(p)]]                                 # noqa: E731
        x = F.conv2d(F.pad(V(S.inp)[:, :3], (3,) * 4, mode="reflect"), pw(bg.conv1.conv.weight), pw(bg.conv1.conv.bias))
        x = st(x * (c64(S.x0) > 0), V(S.x0))
        outs = [x]
        for L in S.layers:
            xp = st(F.pad(x, (1,) * 4, mode="reflect"), V(L.xp))
            x = F.conv2d(xp, pw(L.blk.conv.weight), pw(L.blk.conv.bias), stride=2)
            x = st(x * (c64(L.y) > 0), V(L.y))
            outs.append(x)
        return outs[::-1]
    ref = Ref({n: p for n, p in bg.named_parameters() if not n.startswith("layer4.")}, fwd, [c64(d) for d in dfeats])
    check_params("bg", bg, grads, ref, U_TF32, skip=("layer4.",))


def test_conv_encoder_bwd():
    """conv_encoder_bwd (--use_vae ConvEncoder at crop 256): fc_mu | fc_var weights and biases, the map read in the
    reference's NCHW flatten order, the last InstanceNorm and sn_conv_stack_bwd over the six layers.  TF32 GEMMs."""
    E = _filled(networks.ConvEncoder(_opt(crop_size=256, use_vae=True)), 81)
    gen = torch.Generator().manual_seed(82)
    img = (torch.rand(CFG["batch"], 3, 256, 256, generator=gen) * 2 - 1).to(DEV)
    S = SimpleNamespace()
    with torch.no_grad():
        E.run(img, S)
    dout = torch.randn(CFG["batch"], 512, generator=gen)
    grads = autograd._Grads()
    autograd.conv_encoder_bwd(grads, E, S, dout.to(DEV).view(-1, 1, 1, 512))
    torch.cuda.synchronize()
    names = param_names(E)
    N = CFG["batch"]

    def fwd(P, A):
        V = value(A)
        y = _stack_ref(E, S, names, P, A, 6)
        a = norm(y, (2, 3), A, c64(S.y6)) * lrelu_mask(in_pos(S.y6, S.ss6))
        a = st(a, V(S.a6.view(S.y6.shape)))
        flat = a.reshape(N, -1)
        return [torch.cat([flat @ P["fc_mu.weight"].t() + P["fc_mu.bias"], flat @ P["fc_var.weight"].t() + P["fc_var.bias"]], 1)]
    ref = Ref({n: p for n, p in E.named_parameters()}, fwd, [d64(dout)])
    check_params("ConvEncoder", E, grads, ref, U_TF32)


# ============================================================================================== discriminator


@pytest.mark.parametrize("setting", ["d_step", "g_step", "no_ganFeat_loss"])
def test_discriminator_bwd(setting):
    """_DiscriminatorFn.backward over both scales: _d_scale_bwd per scale (conv_to1_bwd of the logits, in_bwd + SN weight
    gradients + conv_dgrad accumulated into the layer below, the thin conv of model0, thin_dgrad3 into the image) and the
    avgpool3s2_bwd that carries the coarse scale's image gradient to the fine one.  d_step: every parameter gradient and
    the image gradient; g_step: parameters frozen as pix2pix_model freezes them, image gradient only; no_ganFeat_loss: only
    the logits get a gradient.  The conditioning channels get exactly zero.  TF32 gradient GEMMs."""
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import _frozen
    sd = reference_layout_state("D", CFG, 32)
    D = networks.MultiscaleDiscriminator(make_opt(is_train=True, ngf=64, ndf=64, crop_size=CFG["size"],
                                                  no_ganFeat_loss=setting == "no_ganFeat_loss"))
    D.load_state_dict(sd)
    D = D.to(DEV).train()
    gen = torch.Generator().manual_seed(91)
    B, H = CFG["batch"], CFG["size"]
    x = torch.randn(B, 7, H, H, generator=gen) * 0.7
    states = []
    with torch.no_grad():
        result, inv_of = D.run(x.to(DEV), states)
    params = list(D.parameters())
    gouts = []
    for outs in result:
        for j, o in enumerate(outs):
            feat = j < len(outs) - 1
            gouts.append(None if (feat and setting == "no_ganFeat_loss") else torch.randn(o.shape, generator=gen))
    with _frozen(D) if setting == "g_step" else torch.no_grad():
        ctx = SimpleNamespace(netD=D, states=states, inv_of=inv_of, params=params, need_dimg=True,
                              param_grads=any(p.requires_grad for p in params), in_shape=tuple(x.shape))
    assert ctx.param_grads == (setting != "g_step")
    res = autograd._DiscriminatorFn.backward(ctx, *[None if g is None else g.to(DEV) for g in gouts])
    torch.cuda.synchronize()
    dx, pgrads = res[1], res[2:]
    names = [n for n, _ in D.named_parameters()]
    children = [c for _, c in D.named_children()]
    S0, S1 = states

    def fwd(P, A):
        V = value(A)
        outs = []
        xin = P["x"]
        for i, (Dc, S) in enumerate(zip(children, states)):
            pre = "discriminator_%d." % i
            if i:
                xin = st(F.avg_pool2d(xin, 3, 2, 1, count_include_pad=False), V(S.x8)[:, :7])
            f = F.conv2d(xin, P[pre + "model0.0.weight"], P[pre + "model0.0.bias"], stride=2, padding=Dc.padw)
            f = st(f * lrelu_mask(c64(S.f0) > 0), V(S.f0))
            outs.append(f)
            for j, L in enumerate(S.layers):
                n = j + 1
                w = sn_weight(P[pre + "model%d.0.0.weight_orig" % n], L.conv, A)
                raw = st(F.conv2d(f, w, None, stride=L.stride, padding=Dc.padw), V(L.raw))
                f = norm(raw, (2, 3), A, c64(L.raw)) * lrelu_mask(in_pos(L.raw, L.ss))
                f = st(f, V(S.layers[j + 1].f_in if j + 1 < len(S.layers) else S.f_last))
                outs.append(f)
            last = "model%d.0." % Dc.n_layers
            outs.append(F.conv2d(f, P[pre + last + "weight"], P[pre + last + "bias"], padding=Dc.padw))
        keep = [k for k, g in enumerate(gouts) if g is not None]
        return [outs[k] for k in keep]
    leaves = dict(D.named_parameters())
    leaves["x"] = x
    ref = Ref(leaves, fwd, [d64(g) for g in gouts if g is not None])
    tag = "D %s" % setting
    assert float(dx[:, :4].abs().max()) == 0.0   # the image gradient lands in channels 4:7 only
    check(tag, "dx image", dx[:, 4:7], ref.grad["x"][:, 4:7], ref.rabs["x"][:, 4:7], U_TF32)
    if setting == "g_step":
        assert all(g is None for g in pgrads)
        return
    for n, g in zip(names, pgrads):
        assert g is not None, (tag, n)
        check(tag, n, g, ref.grad[n], ref.rabs[n], U_TF32)


# ---------------------------------------------------------------------------------------------- measured ratios
# max |got - ref| / (u R_abs) of every checked tensor, measured on an H100 80GB HBM3 (700 W power limit); k is HEADROOM
# times the value.  Within a case the ratio still differs by tensor: a sum over a few rows (the fc and latent heads) keeps
# its rounding errors, a sum over every pixel of the map (the biases, the weights of high-resolution layers) averages them
# out, so each tensor keeps its own k.
HEADROOM = 4
MEASURED = {
    'mixed16 head_0': {'dx': 1.35, 'conv_0.bias': 4.35e-05, 'conv_0.weight_orig': 5.03, 'conv_1.bias': 3.07e-05,
        'conv_1.weight_orig': 1.74, 'norm_0.mlp_shared.0.weight': 0.0347, 'norm_0.mlp_shared.0.bias': 0.0247,
        'norm_0.mlp_gamma.weight': 11.7, 'norm_0.mlp_gamma.bias': 1.97, 'norm_0.mlp_beta.weight': 3.87,
        'norm_0.mlp_beta.bias': 0.845, 'norm_1.mlp_shared.0.weight': 0.0288, 'norm_1.mlp_shared.0.bias': 0.0288,
        'norm_1.mlp_gamma.weight': 9.13, 'norm_1.mlp_gamma.bias': 1.4, 'norm_1.mlp_beta.weight': 2.91,
        'norm_1.mlp_beta.bias': 0.897},
    'mixed16 G_middle_0': {'dx': 0.465, 'conv_0.bias': 1.45e-05, 'conv_0.weight_orig': 1.2, 'conv_1.bias': 1.53e-05,
        'conv_1.weight_orig': 1, 'norm_0.mlp_shared.0.weight': 0.0318, 'norm_0.mlp_shared.0.bias': 0.0114,
        'norm_0.mlp_gamma.weight': 1.82, 'norm_0.mlp_gamma.bias': 0.764, 'norm_0.mlp_beta.weight': 1.1,
        'norm_0.mlp_beta.bias': 0.369, 'norm_1.mlp_shared.0.weight': 0.022, 'norm_1.mlp_shared.0.bias': 0.00904,
        'norm_1.mlp_gamma.weight': 2.46, 'norm_1.mlp_gamma.bias': 0.474, 'norm_1.mlp_beta.weight': 1.46,
        'norm_1.mlp_beta.bias': 0.372},
    'mixed16 G_middle_1': {'dx': 0.546, 'conv_0.bias': 6.91e-06, 'conv_0.weight_orig': 0.522, 'conv_1.bias': 6.55e-06,
        'conv_1.weight_orig': 0.542, 'norm_0.mlp_shared.0.weight': 0.0169, 'norm_0.mlp_shared.0.bias': 0.00585,
        'norm_0.mlp_gamma.weight': 0.769, 'norm_0.mlp_gamma.bias': 0.252, 'norm_0.mlp_beta.weight': 0.46,
        'norm_0.mlp_beta.bias': 0.155, 'norm_1.mlp_shared.0.weight': 0.0139, 'norm_1.mlp_shared.0.bias': 0.012,
        'norm_1.mlp_gamma.weight': 0.604, 'norm_1.mlp_gamma.bias': 0.202, 'norm_1.mlp_beta.weight': 0.347,
        'norm_1.mlp_beta.bias': 0.159},
    'mixed16 up_0': {'dx': 0.72, 'dbf': 0, 'conv_0.bias': 4.51e-06, 'conv_0.weight_orig': 0.39, 'conv_1.bias': 4.69e-06,
        'conv_1.weight_orig': 0.41, 'conv_s.weight_orig': 0.306, 'norm_0.mlp_shared.0.weight': 0.0186,
        'norm_0.mlp_shared.0.bias': 0.00895, 'norm_0.mlp_gamma.weight': 0.413, 'norm_0.mlp_gamma.bias': 0.187,
        'norm_0.mlp_beta.weight': 0.268, 'norm_0.mlp_beta.bias': 0.0901, 'norm_1.mlp_shared.0.weight': 0.0409,
        'norm_1.mlp_shared.0.bias': 0.00459, 'norm_1.mlp_gamma.weight': 0.549, 'norm_1.mlp_gamma.bias': 0.148,
        'norm_1.mlp_beta.weight': 0.294, 'norm_1.mlp_beta.bias': 0.148, 'norm_s.mlp_shared.0.weight': 0.0143,
        'norm_s.mlp_shared.0.bias': 0.00328, 'norm_s.mlp_gamma.weight': 0.395, 'norm_s.mlp_gamma.bias': 0.13,
        'norm_s.mlp_beta.weight': 0.224, 'norm_s.mlp_beta.bias': 0.0942},
    'mixed16 up_1': {'dx': 0.78, 'dbf': 0, 'conv_0.bias': 3.63e-06, 'conv_0.weight_orig': 0.281, 'conv_1.bias': 1.89e-06,
        'conv_1.weight_orig': 0.215, 'conv_s.weight_orig': 0.14, 'norm_0.mlp_shared.0.weight': 0.0534,
        'norm_0.mlp_shared.0.bias': 0.00473, 'norm_0.mlp_gamma.weight': 0.282, 'norm_0.mlp_gamma.bias': 0.0981,
        'norm_0.mlp_beta.weight': 0.205, 'norm_0.mlp_beta.bias': 0.0705, 'norm_1.mlp_shared.0.weight': 0.0221,
        'norm_1.mlp_shared.0.bias': 0.0165, 'norm_1.mlp_gamma.weight': 0.601, 'norm_1.mlp_gamma.bias': 0.0624,
        'norm_1.mlp_beta.weight': 0.289, 'norm_1.mlp_beta.bias': 0.0665, 'norm_s.mlp_shared.0.weight': 0.0185,
        'norm_s.mlp_shared.0.bias': 0.00593, 'norm_s.mlp_gamma.weight': 0.23, 'norm_s.mlp_gamma.bias': 0.0708,
        'norm_s.mlp_beta.weight': 0.113, 'norm_s.mlp_beta.bias': 0.0466},
    'mixed16 up_2': {'dx': 0.918, 'dbf': 0, 'conv_0.bias': 2.85e-06, 'conv_0.weight_orig': 0.1, 'conv_1.bias': 1.02e-06,
        'conv_1.weight_orig': 0.0879, 'conv_s.weight_orig': 0.0722, 'norm_0.mlp_shared.0.weight': 0.0499,
        'norm_0.mlp_shared.0.bias': 0.00527, 'norm_0.mlp_gamma.weight': 0.0747, 'norm_0.mlp_gamma.bias': 0.0417,
        'norm_0.mlp_beta.weight': 0.0655, 'norm_0.mlp_beta.bias': 0.0321, 'norm_1.mlp_shared.0.weight': 0.0344,
        'norm_1.mlp_shared.0.bias': 0.00425, 'norm_1.mlp_gamma.weight': 0.0469, 'norm_1.mlp_gamma.bias': 0.0416,
        'norm_1.mlp_beta.weight': 0.0402, 'norm_1.mlp_beta.bias': 0.0362, 'norm_s.mlp_shared.0.weight': 0.0462,
        'norm_s.mlp_shared.0.bias': 0.00722, 'norm_s.mlp_gamma.weight': 0.133, 'norm_s.mlp_gamma.bias': 0.0359,
        'norm_s.mlp_beta.weight': 0.0608, 'norm_s.mlp_beta.bias': 0.0187},
    'mixed16 up_3': {'dx': 0.894, 'dbf': 0, 'conv_0.bias': 2.19e-06, 'conv_0.weight_orig': 0.0533, 'conv_1.bias': 3.91e-07,
        'conv_1.weight_orig': 0.0438, 'conv_s.weight_orig': 0.0338, 'norm_0.mlp_shared.0.weight': 0.0475,
        'norm_0.mlp_shared.0.bias': 0.00277, 'norm_0.mlp_gamma.weight': 0.0275, 'norm_0.mlp_gamma.bias': 0.0216,
        'norm_0.mlp_beta.weight': 0.0232, 'norm_0.mlp_beta.bias': 0.014, 'norm_1.mlp_shared.0.weight': 0.0513,
        'norm_1.mlp_shared.0.bias': 0.016, 'norm_1.mlp_gamma.weight': 0.0466, 'norm_1.mlp_gamma.bias': 0.017,
        'norm_1.mlp_beta.weight': 0.0413, 'norm_1.mlp_beta.bias': 0.0159, 'norm_s.mlp_shared.0.weight': 0.0402,
        'norm_s.mlp_shared.0.bias': 0.0027, 'norm_s.mlp_gamma.weight': 0.0248, 'norm_s.mlp_gamma.bias': 0.0161,
        'norm_s.mlp_beta.weight': 0.0194, 'norm_s.mlp_beta.bias': 0.0131},
    'tf32 G_middle_0': {'dx': 0.72, 'conv_0.bias': 0.000102, 'conv_0.weight_orig': 1.39, 'conv_1.bias': 0.000122,
        'conv_1.weight_orig': 1.4, 'norm_0.mlp_shared.0.weight': 0.0658, 'norm_0.mlp_shared.0.bias': 0.0162,
        'norm_0.mlp_gamma.weight': 2.18, 'norm_0.mlp_gamma.bias': 0.936, 'norm_0.mlp_beta.weight': 1.29,
        'norm_0.mlp_beta.bias': 0.553, 'norm_1.mlp_shared.0.weight': 0.0289, 'norm_1.mlp_shared.0.bias': 0.0113,
        'norm_1.mlp_gamma.weight': 2.86, 'norm_1.mlp_gamma.bias': 0.544, 'norm_1.mlp_beta.weight': 1.31,
        'norm_1.mlp_beta.bias': 0.442},
    'tf32 up_1': {'dx': 1.19, 'dbf': 0, 'conv_0.bias': 2.88e-05, 'conv_0.weight_orig': 0.501, 'conv_1.bias': 1.51e-05,
        'conv_1.weight_orig': 0.296, 'conv_s.weight_orig': 0.219, 'norm_0.mlp_shared.0.weight': 0.0708,
        'norm_0.mlp_shared.0.bias': 0.00803, 'norm_0.mlp_gamma.weight': 0.534, 'norm_0.mlp_gamma.bias': 0.187,
        'norm_0.mlp_beta.weight': 0.332, 'norm_0.mlp_beta.bias': 0.148, 'norm_1.mlp_shared.0.weight': 0.0475,
        'norm_1.mlp_shared.0.bias': 0.0294, 'norm_1.mlp_gamma.weight': 0.455, 'norm_1.mlp_gamma.bias': 0.107,
        'norm_1.mlp_beta.weight': 0.267, 'norm_1.mlp_beta.bias': 0.0905, 'norm_s.mlp_shared.0.weight': 0.0263,
        'norm_s.mlp_shared.0.bias': 0.0069, 'norm_s.mlp_gamma.weight': 0.236, 'norm_s.mlp_gamma.bias': 0.0995,
        'norm_s.mlp_beta.weight': 0.119, 'norm_s.mlp_beta.bias': 0.0765},
    'mixed16_grad16_gb head_0': {'dx': 0.159, 'conv_0.bias': 7.06e-05, 'conv_0.weight_orig': 0.523, 'conv_1.bias': 3.07e-05,
        'conv_1.weight_orig': 0.419, 'norm_0.mlp_shared.0.weight': 0.0255, 'norm_0.mlp_shared.0.bias': 0.0136,
        'norm_0.mlp_gamma.weight': 1.67, 'norm_0.mlp_gamma.bias': 0.216, 'norm_0.mlp_beta.weight': 1.26,
        'norm_0.mlp_beta.bias': 0.154, 'norm_1.mlp_shared.0.weight': 0.0242, 'norm_1.mlp_shared.0.bias': 0.0119,
        'norm_1.mlp_gamma.weight': 1.22, 'norm_1.mlp_gamma.bias': 0.159, 'norm_1.mlp_beta.weight': 1.1,
        'norm_1.mlp_beta.bias': 0.107},
    'mixed16_grad16_gb up_0': {'dx': 0.13, 'dbf': 0, 'conv_0.bias': 4.14e-06, 'conv_0.weight_orig': 0.113,
        'conv_1.bias': 4.69e-06, 'conv_1.weight_orig': 0.12, 'conv_s.weight_orig': 0.108, 'norm_0.mlp_shared.0.weight': 0.0165,
        'norm_0.mlp_shared.0.bias': 0.00386, 'norm_0.mlp_gamma.weight': 0.211, 'norm_0.mlp_gamma.bias': 0.0397,
        'norm_0.mlp_beta.weight': 0.147, 'norm_0.mlp_beta.bias': 0.0185, 'norm_1.mlp_shared.0.weight': 0.0228,
        'norm_1.mlp_shared.0.bias': 0.00334, 'norm_1.mlp_gamma.weight': 0.309, 'norm_1.mlp_gamma.bias': 0.0236,
        'norm_1.mlp_beta.weight': 0.207, 'norm_1.mlp_beta.bias': 0.0191, 'norm_s.mlp_shared.0.weight': 0.0168,
        'norm_s.mlp_shared.0.bias': 0.00236, 'norm_s.mlp_gamma.weight': 0.243, 'norm_s.mlp_gamma.bias': 0.0286,
        'norm_s.mlp_beta.weight': 0.178, 'norm_s.mlp_beta.bias': 0.0246},
    'ImageEncoder3': {'layer1.weight': 0.0454, 'layer1.bias': 0.00852, 'layer2.weight': 0.0201, 'layer2.bias': 0.00208,
        'layer3.weight': 0.0378, 'layer3.bias': 0.00225, 'layer4.weight': 0.0646, 'layer4.bias': 0.000903,
        'layer5.weight': 0.185, 'layer5.bias': 2.06e-06},
    'ImageEncoder2 pick=True': {'layer1.0.weight_orig': 0.00258, 'layer2.0.weight_orig': 0.000659,
        'layer3.0.weight_orig': 0.000689, 'layer4.0.weight_orig': 0.00087, 'layer5.0.weight_orig': 0.00289},
    'ImageEncoder2 pick=False': {'layer1.0.weight_orig': 0.0024, 'layer2.0.weight_orig': 0.000684,
        'layer3.0.weight_orig': 0.000708, 'layer4.0.weight_orig': 0.000961, 'layer5.0.weight_orig': 0.00199},
    'ImageEncoder': {'layer1.0.weight_orig': 0.00163, 'layer2.0.weight_orig': 0.000474, 'layer3.0.weight_orig': 0.000384,
        'layer4.0.weight_orig': 0.000453, 'layer5.0.weight_orig': 0.00133, 'fc.weight': 3.47, 'fc.bias': 1.86},
    'vae head': {'dW': 3.68, 'db': 1.85, 'dz': 0.0754},
    'bg': {'conv1.conv.weight': 0.00442, 'conv1.conv.bias': 0.00219, 'layer1.conv.weight': 0.246, 'layer1.conv.bias': 0.0177,
        'layer2.conv.weight': 1.78, 'layer2.conv.bias': 0.316, 'layer3.conv.weight': 1.94, 'layer3.conv.bias': 0.477},
    'ConvEncoder': {'layer1.0.weight_orig': 0.00175, 'layer2.0.weight_orig': 0.000439, 'layer3.0.weight_orig': 0.000511,
        'layer4.0.weight_orig': 0.000541, 'layer5.0.weight_orig': 0.00069, 'layer6.0.weight_orig': 0.00184,
        'fc_mu.weight': 3.75, 'fc_mu.bias': 0.00012, 'fc_var.weight': 3.81, 'fc_var.bias': 0.000119},
    'D d_step': {'dx image': 0.259, 'discriminator_0.model0.0.weight': 0.0363, 'discriminator_0.model0.0.bias': 0.0123,
        'discriminator_0.model1.0.0.weight_orig': 0.0984, 'discriminator_0.model2.0.0.weight_orig': 0.206,
        'discriminator_0.model3.0.0.weight_orig': 0.218, 'discriminator_0.model4.0.weight': 2.99e-05,
        'discriminator_0.model4.0.bias': 5.88e-06, 'discriminator_1.model0.0.weight': 0.0733,
        'discriminator_1.model0.0.bias': 0.0259, 'discriminator_1.model1.0.0.weight_orig': 0.215,
        'discriminator_1.model2.0.0.weight_orig': 0.421, 'discriminator_1.model3.0.0.weight_orig': 0.365,
        'discriminator_1.model4.0.weight': 4.35e-05, 'discriminator_1.model4.0.bias': 1.83e-06},
    'D g_step': {'dx image': 0.259},
    'D no_ganFeat_loss': {'dx image': 0.325, 'discriminator_0.model0.0.weight': 0.0394,
        'discriminator_0.model0.0.bias': 0.0166, 'discriminator_0.model1.0.0.weight_orig': 0.114,
        'discriminator_0.model2.0.0.weight_orig': 0.252, 'discriminator_0.model3.0.0.weight_orig': 0.189,
        'discriminator_0.model4.0.weight': 2.72e-05, 'discriminator_0.model4.0.bias': 4.83e-06,
        'discriminator_1.model0.0.weight': 0.0931, 'discriminator_1.model0.0.bias': 0.0269,
        'discriminator_1.model1.0.0.weight_orig': 0.236, 'discriminator_1.model2.0.0.weight_orig': 0.485,
        'discriminator_1.model3.0.0.weight_orig': 0.395, 'discriminator_1.model4.0.weight': 6.13e-05,
        'discriminator_1.model4.0.bias': 8.54e-07},
}
