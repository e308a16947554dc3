"""Training path: hand-written backward passes wired into torch.autograd as three Functions
(generator, multiscale discriminator, the --use_vae ConvEncoder); the generator's reference-image encoder is reached through
its backward_nhwc method.  Forward = the networks' ONE forward implementation (`SPADEBGenerator.run`,
`MultiscaleDiscriminator.run`) in "save" mode: the same kernels and operand formats as inference (precision.py), which
additionally keep the fp32 value of every tensor the gradient GEMMs need (read as TF32 by the wgrad / dgrad kernels);
backward = explicit reverse pass over the saved per-block state:

    conv  : dW = mg_conv_wgrad (mma.sync, MN-major, split-K);  dX = mg_conv_igemm on dY with flipped sub-kernels
    SPADE : mg_spade_bwd (dgamma|dbeta operand, dxhat, BN sums)  ->  gamma/beta GEMM wgrad + dgrad  ->  thin wgrad
    BN/IN : mg_bn_bwd_apply / mg_in_bwd (statistics all-reduced across ranks like the forward ones)
    SN    : mg_spectral_norm_bwd (u, v constants, as torch's spectral_norm autograd)

What is saved per SPADE: h (conv operand), 1+gamma, the normalisation vectors; `actv` is recomputed.
"""
from types import SimpleNamespace

import torch

from .. import ops, precision
from .sync_batchnorm import allreduce_sums

_RELU, _LRELU, _NONE = ops.ACT_RELU, ops.ACT_LRELU, ops.ACT_NONE


def _nhwc(g):
    """NCHW-shaped gradient (any strides) -> contiguous NHWC tensor that this backward owns (it is
    used as an accumulation target, so never alias the tensor autograd handed in)."""
    t = g.permute(0, 2, 3, 1)
    return t.clone(memory_format=torch.contiguous_format)


class _Grads:
    """param -> accumulated gradient."""

    def __init__(self):
        self.d = {}

    def add(self, p, g):
        if p is None or g is None:
            return
        g = g.reshape(p.shape)
        k = id(p)
        self.d[k] = g if k not in self.d else self.d[k] + g

    def get(self, p):
        return self.d.get(id(p))


def _thin_wt_to_oihw(dwt, kh, kw, cin):
    """[kh*kw][CinP][Cout] -> [Cout, cin, kh, kw]."""
    cp, co = dwt.shape[1], dwt.shape[2]
    return dwt.view(kh, kw, cp, co).permute(3, 2, 0, 1)[:, :cin].contiguous()


# =============================================================================================== conv helpers
def _conv_weight(conv, inv_of):
    """(w_oihw source, inv_sigma or None, is_sn)."""
    if hasattr(conv, "weight_orig"):
        return conv.weight_orig, inv_of[conv], True
    return conv.weight, None, False


def _conv_param_grads(G, conv, inv_of, dy, a_operand, kh, kw, stride, pad, with_bias=True, dz_for_bias=None, dy16=None, a16=None,
                      bias_sum=None):
    """Weight (+bias) gradients of an implicit-GEMM conv; dy: [N,OH,OW,Cout], a_operand: its fp32 input.
    dy16 / a16: bf16 copies (both given -> bf16 weight-gradient GEMM)."""
    w, isg, is_sn = _conv_weight(conv, inv_of)
    if dy16 is not None and a16 is None and a_operand.shape[-1] % 64 == 0:
        a16 = ops.cvt16(a_operand, ops.BF16)
    if dy16 is not None and a16 is not None:
        dwp = ops.conv_wgrad16(dy16, a16, kh, kw, stride, pad)
    else:
        dwp = ops.conv_wgrad(dy, a_operand, kh, kw, stride, pad)
    dwt = ops.unpack_wgrad(dwp, tuple(w.shape))
    if is_sn:
        G.add(w, ops.spectral_norm_bwd(dwt, w.detach(), conv.weight_u, conv.weight_v, isg))
    else:
        G.add(w, dwt)
    if with_bias and getattr(conv, "bias", None) is not None:
        G.add(conv.bias, bias_sum if bias_sum is not None else ops.chan_sum(dz_for_bias if dz_for_bias is not None else dy))


# =============================================================================================== SPADE + conv
def _spade_conv_bwd(G, blk, S, conv, inv_of, dy, k, pad, seg4):
    """Backward of conv(act(SPADE(src))) given dy; returns (dxhat, sums) for the BN backward of `src`."""
    # bf16 gradient GEMMs: dY's bf16 copy and (for convs with a bias) its channel sums come out of one pass over dY
    dy16 = bias_sum = None
    if precision.conv_grad_fmt() == ops.BF16 and dy.shape[-1] % 64 == 0:
        if getattr(conv, "bias", None) is not None:
            bias_sum, dy16 = ops.chan_sum_cvt16(dy)
        else:
            dy16 = ops.cvt16(dy, ops.BF16)
    _conv_param_grads(G, conv, inv_of, dy, S.h, k, k, 1, pad, dy16=dy16, a16=getattr(S, "h16", None), bias_sum=bias_sum)
    w, isg, _ = _conv_weight(conv, inv_of)
    dh = ops.conv_dgrad(dy, w.detach(), S.hw, 1, pad, inv_sigma=isg, dy16=dy16)
    del dy16
    gfmt = precision.grad_fmt()
    dgb, dxhat, sums, bsum = ops.spade_bwd(dh, S.h, S.g1, S.src, S.shift, S.ns, S.nh, S.act, dgb_fmt=gfmt)
    del dh
    sp = S.sp
    c = S.src.shape[-1]
    wdg = ops.pack_weight_dgrad_gb(sp.mlp_gamma.weight.detach(), sp.mlp_beta.weight.detach())
    if gfmt == ops.TF32:
        actv = ops.mlp_shared(seg4, S.wsh, sp.mlp_shared[0].bias.detach(), seg_resize=S.R, act=_RELU, round_out=True, out_hw=S.hw)
        dwp = ops.conv_wgrad(dgb, actv, 3, 3, 1, 1)
        dactv = ops.conv_igemm(dgb, wdg, 128, 3, 3, 1, 1)
    else:
        actv, actv16, _ = ops.mlp_shared(seg4, S.wsh, sp.mlp_shared[0].bias.detach(), seg_resize=S.R, act=_RELU, out_hw=S.hw,
                                         out16=(gfmt, False))
        dwp = ops.conv_wgrad16(dgb, actv16, 3, 3, 1, 1)
        del actv16
        dactv = ops.conv_igemm(dgb, ops.cvt16(wdg, gfmt), 128, 3, 3, 1, 1, a_fmt=gfmt)
    dwg, dwb = ops.unpack_wgrad_gb(dwp, c, 128)
    G.add(sp.mlp_gamma.weight, dwg)
    G.add(sp.mlp_beta.weight, dwb)
    G.add(sp.mlp_gamma.bias, bsum[:c].float())
    G.add(sp.mlp_beta.bias, bsum[c:].float())
    del dgb
    # ReLU backward of mlp_shared and its bias gradient are fused into the weight-gradient kernel: d actv is read once
    dwt, db = ops.thin_wgrad(seg4, dactv, 3, 3, 1, 1, seg_resize=S.R, in_hw=S.hw, relu_src=actv, want_bias=True)
    del dactv, actv
    G.add(sp.mlp_shared[0].weight, _thin_wt_to_oihw(dwt, 3, 3, 4))
    G.add(sp.mlp_shared[0].bias, db)
    return dxhat, sums, allreduce_sums(sums, dxhat.numel() // c)


# =============================================================================================== SPADEResnetBlock
def block_bwd(G, blk, S, dout, seg4, inv_of):
    """-> (dx wrt the block input (pre-upsample), dbf wrt the blended background feature or None)."""
    dbf = None
    if S.blend is not None:
        _, hair, back, ms = S.blend
        dy, dbf = ops.blend_bwd(dout, hair, back, ms)
    else:
        dy = dout
    dxhat1, sums1, cnt1 = _spade_conv_bwd(G, blk, S.sp1, blk.conv_1, inv_of, dy, 3, 1, seg4)
    ddx = ops.bn_bwd_apply(dxhat1, S.dx, 0, S.sp1.ns, S.sp1.nh, sums1, cnt1)
    del dxhat1
    dxhat0, sums0, cnt0 = _spade_conv_bwd(G, blk, S.sp0, blk.conv_0, inv_of, ddx, 3, 1, seg4)
    del ddx
    dx = ops.bn_bwd_apply(dxhat0, S.x, S.xs, S.sp0.ns, S.sp0.nh, sums0, cnt0)
    del dxhat0
    if blk.learned_shortcut:
        dxhat_s, sums_s, cnt_s = _spade_conv_bwd(G, blk, S.sps, blk.conv_s, inv_of, dy, 1, 0, seg4)
        ops.bn_bwd_apply(dxhat_s, S.x, S.xs, S.sps.ns, S.sps.nh, sums_s, cnt_s, dx=dx)
    else:
        ops.bn_bwd_apply(dy, S.x, S.xs, None, None, None, 1, dx=dx)   # identity shortcut through the upsample
    return dx, dbf


# =============================================================================================== encoders
def fc_bwd(G, fc, S, dout):
    d = ops.resize_bilinear_bwd(dout, S.mhw) if (dout.shape[1], dout.shape[2]) != S.mhw else dout
    d = ops.masked_mean_bcast_bwd(d, S.mref, S.mtag)
    dy = ops.in_bwd(d, S.y5, S.ss6, _LRELU)
    for L in reversed(S.layers):
        dz = ops.act_bwd(dy, None, _NONE, pm1=L.upd, pm2=L.ratio, round_tf32=True)   # d(acc) of (acc*ratio + b)*upd
        G.add(L.layer.bias, ops.chan_sum(ops.act_bwd(dy, None, _NONE, pm1=L.upd)))
        G.add(L.layer.weight, ops.unpack_wgrad(ops.conv_wgrad(dz, L.a, 3, 3, 2, 1), tuple(L.layer.weight.shape)))
        da = ops.conv_dgrad(dz, L.layer.weight.detach(), (L.a.shape[1], L.a.shape[2]), 2, 1)
        dy = ops.in_bwd(da, L.y_in, L.ss, _LRELU, pmul=L.pm_in)
    dz = ops.act_bwd(dy, None, _NONE, pm1=S.l1.upd, pm2=S.l1.ratio)
    G.add(fc.layer1.bias, ops.chan_sum(ops.act_bwd(dy, None, _NONE, pm1=S.l1.upd)))
    dwt1 = ops.thin_wgrad(S.x0, dz, 3, 3, 2, 1)
    G.add(fc.layer1.weight, _thin_wt_to_oihw(dwt1, 3, 3, 3))


def bg_bwd(G, bg, S, dfeats):
    """dfeats: grads of [x3, x2, x1, x0] (from the four background blends)."""
    d_list = dfeats[::-1]   # [dx0, dx1, dx2, dx3]
    d = d_list[3]
    for i in (2, 1, 0):
        L = S.layers[i]
        dz = ops.act_bwd(d, L.y, _RELU, round_tf32=True)
        G.add(L.blk.conv.bias, ops.chan_sum(dz))
        G.add(L.blk.conv.weight, ops.unpack_wgrad(ops.conv_wgrad(dz, L.xp, 4, 4, 2, 0), tuple(L.blk.conv.weight.shape)))
        dxp = ops.conv_dgrad(dz, L.blk.conv.weight.detach(), (L.xp.shape[1], L.xp.shape[2]), 2, 0)
        d = ops.reflect_pad_bwd(dxp, 1, dx=d_list[i])
    dz0 = ops.act_bwd(d, S.x0, _RELU)
    G.add(bg.conv1.conv.bias, ops.chan_sum(dz0))
    dwt1 = ops.thin_wgrad(S.inp, dz0, 7, 7, 1, 3, pad_mode=1)
    G.add(bg.conv1.conv.weight, _thin_wt_to_oihw(dwt1, 7, 7, 3))


def latent_bwd(G, fc, S, dx):
    """Backward of encoder.latent_head, x = view(z W^T + b): the --use_vae head (generator.py:110-116) and ImageEncoder's fc
    (encoder.py:99-101), given dx [N,sh,sw,C] NHWC; returns dz [N, K].  The weight and bias gradients read dx in the
    reference's NCHW row order (one transpose of the N x C*sh*sw gradient), so they come out in fc.weight's own layout.  They
    are one weight-gradient GEMM over the N rows: z is extended by a column of ones (the bias) and 31 zeros (the GEMM's
    32-column granule), so dW | db = dY^T [z | 1 | 0] (the per-channel sum kernels take at most 4096 channels; the head has
    C*sh*sw).  dz is the 1x1 data-gradient GEMM on the permuted weight the forward packed (S.wp)."""
    N = dx.shape[0]
    K = dx[0].numel()
    dy_ref = ops.nhwc_to_nchw(dx).view(N, 1, 1, K)
    zd = S.z4.shape[-1]
    za = torch.cat([S.z4.view(N, zd), torch.ones((N, 1), device=dx.device), torch.zeros((N, 31), device=dx.device)], 1)
    dwa = ops.conv_wgrad(dy_ref, za.view(N, 1, 1, zd + 32), 1, 1, 1, 0)
    G.add(fc.weight, dwa[:, :zd])
    G.add(fc.bias, dwa[:, zd])
    return ops.conv_dgrad(dx.view(N, 1, 1, K), S.wp.view(K, -1, 1, 1), (1, 1), 1, 0).view(N, -1)


# =============================================================================================== generator Function
class _GeneratorFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, netG, z, input_ref, orient_mask, image_ref, input_tag, noise, image_tag, *params):
        st = SimpleNamespace()
        out = netG.run(input_ref, orient_mask, image_ref, input_tag, noise, image_tag, st, z=z)
        ctx.netG, ctx.seg4, ctx.inv_of, ctx.saved, ctx.Sfc, ctx.Sbg, ctx.x_last, ctx.out = \
            netG, st.seg4, st.inv_of, st.saved, st.Sfc, st.Sbg, st.x_last, st.out
        ctx.params = params
        return out

    @staticmethod
    def backward(ctx, dout):
        netG, seg4, inv_of = ctx.netG, ctx.seg4, ctx.inv_of
        G = _Grads()
        red = getattr(netG, "_grad_reducer", None)   # data-parallel: stages are all-reduced while later stages compute
        if red is not None:
            red.begin(ctx.params)
        dx, dw, db = ops.conv_img_bwd(dout.contiguous(), ctx.out, ctx.x_last, netG.conv_img.weight.detach())
        G.add(netG.conv_img.weight, dw)
        G.add(netG.conv_img.bias, db)
        names = netG._blocks
        stage_of = netG.GRAD_STAGE_AFTER_BLOCK
        dfeats = [None] * 4
        for idx in range(6, -1, -1):
            blk = getattr(netG, names[idx])
            dx, dbf = block_bwd(G, blk, ctx.saved[idx], dx, seg4, inv_of)
            ctx.saved[idx] = None
            if idx >= 3:
                dfeats[idx - 3] = dbf
            if red is not None and names[idx] in stage_of:
                red.reduce_stage(stage_of[names[idx]], G.get)
        dz = None
        if getattr(netG.opt, "use_vae", False):
            dz = latent_bwd(G, netG.fc, ctx.Sfc, dx)
            if not ctx.needs_input_grad[1]:
                dz = None
        else:
            netG.fc.backward_nhwc(G, ctx.Sfc, dx)
        bg_bwd(G, netG.backgroud_enc, ctx.Sbg, dfeats)
        ctx.saved = ctx.Sfc = ctx.Sbg = None
        if red is not None:
            red.reduce_stage(len(red.stages) - 1, G.get)
            return (None, dz) + (None,) * 6 + red.finish(ctx.params, G.get)
        return (None, dz) + (None,) * 6 + tuple(G.get(p) for p in ctx.params)


def generator_forward_autograd(netG, input_ref, orient_mask, image_ref, input_tag, noise, image_tag, z=None):
    params = [p for p in netG.parameters()]
    return _GeneratorFn.apply(netG, z, input_ref, orient_mask, image_ref, input_tag, noise, image_tag, *params)


# =============================================================================================== ConvEncoder Function
def sn_conv_stack_bwd(G, convs, S, dy):
    """Parameter gradients of encoder.SNConvStack.run_stack given dy, the TF32-rounded gradient of its output: its SN conv +
    InstanceNorm + LeakyReLU layers in reverse, as _d_scale_bwd does for the discriminator's convs.  convs: the stack's
    convs(); S: the namespace run_stack filled."""
    for L in reversed(S.layers):
        _conv_param_grads(G, L.conv, S.inv_of, dy, L.a, 3, 3, 2, 1, with_bias=False)
        w, isg, _ = _conv_weight(L.conv, S.inv_of)
        da = ops.conv_dgrad(dy, w.detach(), (L.a.shape[1], L.a.shape[2]), 2, 1, inv_sigma=isg)
        dy = ops.in_bwd(da, L.y_in, L.ss, _LRELU, round_tf32=L is not S.layers[0])
    conv1 = convs[0]
    w1, isg1, is_sn = _conv_weight(conv1, S.inv_of)
    dwt = _thin_wt_to_oihw(ops.thin_wgrad(S.x0, dy, 3, 3, 2, 1), 3, 3, 3)
    G.add(w1, ops.spectral_norm_bwd(dwt, w1.detach(), conv1.weight_u, conv1.weight_v, isg1) if is_sn else dwt)


def conv_encoder_bwd(G, E, S, dout):
    """Parameter gradients of ConvEncoder.run given dout = d(mu | logvar) [N,1,1,512]: fc_mu | fc_var weight and bias, then the
    six layers of the stack (sn_conv_stack_bwd)."""
    N = dout.shape[0]
    dwf = ops.conv_wgrad(dout, S.a6, 1, 1, 1, 0)                  # [512, 16C], columns in the map's NHWC order
    c = S.y6.shape[-1]
    dwf = dwf.view(512, 16, c).transpose(1, 2).reshape(512, 16 * c)
    G.add(E.fc_mu.weight, dwf[:256])
    G.add(E.fc_var.weight, dwf[256:])
    db = ops.chan_sum(dout)
    G.add(E.fc_mu.bias, db[:256])
    G.add(E.fc_var.bias, db[256:])
    da = ops.conv_dgrad(dout, E.fc_weight(), (1, 1), 1, 0).view(S.y6.shape)
    sn_conv_stack_bwd(G, E.convs(), S, ops.in_bwd(da, S.y6, S.ss6, _LRELU, round_tf32=True))


class _ConvEncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, netE, image, *params):
        st = SimpleNamespace()
        mu, logvar = netE.run(image, st)
        ctx.netE, ctx.st, ctx.params = netE, st, params
        return mu, logvar

    @staticmethod
    def backward(ctx, dmu, dlogvar):
        netE = ctx.netE
        G = _Grads()
        red = getattr(netE, "_grad_reducer", None)
        if red is not None:
            red.begin(ctx.params)
        N = ctx.st.y6.shape[0]
        dmu = torch.zeros((N, 256), device=ctx.st.y6.device) if dmu is None else dmu
        dlogvar = torch.zeros((N, 256), device=ctx.st.y6.device) if dlogvar is None else dlogvar
        dout = torch.cat([dmu, dlogvar], dim=1).float().view(N, 1, 1, 512)
        conv_encoder_bwd(G, netE, ctx.st, dout)
        ctx.st = None
        if red is not None:
            red.reduce_stage(0, G.get)
            return (None, None) + red.finish(ctx.params, G.get)
        return (None, None) + tuple(G.get(p) for p in ctx.params)


def conv_encoder_forward_autograd(netE, image):
    return _ConvEncoderFn.apply(netE, image, *netE.parameters())


# =============================================================================================== discriminator Function
def _d_scale_bwd(G, D, S, douts, inv_of, need_dimg, param_grads):
    """douts: list of NHWC grads (or None) for [f0..f3, logits]; returns dimg NCHW [B,3,H,W] or None."""
    nl = D.n_layers
    df = douts[nl - 1]
    if douts[nl] is not None:
        dxl, dw, db = ops.conv_to1_bwd(douts[nl], S.f_last, S.last.weight.detach(), D.padw, dx=df, want_dx=True)
        df = dxl
        if param_grads:
            G.add(S.last.weight, dw)
            G.add(S.last.bias, db)
    for n in range(nl - 1, 0, -1):
        L = S.layers[n - 1]
        below = douts[n - 1]
        if df is None:
            df = below
            continue
        draw = ops.in_bwd(df, L.raw, L.ss, _LRELU, round_tf32=True)
        w, isg, _ = _conv_weight(L.conv, inv_of)
        if param_grads:
            _conv_param_grads(G, L.conv, inv_of, draw, L.f_in, 4, 4, L.stride, D.padw, with_bias=False)
        df = ops.conv_dgrad(draw, w.detach(), (L.f_in.shape[1], L.f_in.shape[2]), L.stride, D.padw, inv_sigma=isg,
                            out=below, accumulate=below is not None)
    if df is None:
        return None
    conv0 = D.model0[0]
    dz0 = ops.act_bwd(df, S.f0, _LRELU)
    if param_grads:
        dwt0 = ops.thin_wgrad(S.x8, dz0, 4, 4, 2, D.padw)
        G.add(conv0.weight, _thin_wt_to_oihw(dwt0, 4, 4, conv0.weight.shape[1]))
        G.add(conv0.bias, ops.chan_sum(dz0))
    if not need_dimg:
        return None
    B, H, W, _ = S.x8.shape
    dimg = torch.zeros((B, 3, H, W), device=dz0.device, dtype=torch.float32)
    ops.thin_dgrad3(dz0, S.wt0, dimg, 4, 4, 2, D.padw, 4)
    return dimg


class _DiscriminatorFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, netD, x_nchw, *params):
        states = []
        result, inv_of = netD.run(x_nchw, states)
        flat = [o for outs in result for o in outs]
        ctx.netD, ctx.states, ctx.inv_of, ctx.params = netD, states, inv_of, params
        ctx.need_dimg = x_nchw.requires_grad
        ctx.param_grads = any(p.requires_grad for p in params)
        ctx.in_shape = tuple(x_nchw.shape)
        return tuple(flat)

    @staticmethod
    def backward(ctx, *gouts):
        netD = ctx.netD
        G = _Grads()
        children = [D for _, D in netD.named_children()]
        per = children[0].n_layers + 1
        dimg_total = None
        red = getattr(netD, "_grad_reducer", None) if ctx.param_grads else None
        if red is not None:
            red.begin(ctx.params)
        for i in range(len(children) - 1, -1, -1):
            douts = [(_nhwc(g) if g is not None else None) for g in gouts[i * per:(i + 1) * per]]
            dimg = _d_scale_bwd(G, children[i], ctx.states[i], douts, ctx.inv_of, ctx.need_dimg, ctx.param_grads)
            if red is not None:
                red.reduce_stage(len(children) - 1 - i, G.get)   # stage order = backward order (coarsest scale first)
            if ctx.need_dimg and dimg is not None:
                if dimg_total is None:
                    dimg_total = dimg
                else:
                    # gradient of the finer scale's avg-pooled input (dimg_total is at the coarser scale)
                    fine = torch.zeros((dimg.shape[0], dimg.shape[2], dimg.shape[3], 4), device=dimg.device)
                    ops.avgpool3s2_bwd(ops.nchw_to_nhwc(dimg_total, 4), fine)
                    dimg_total = dimg + ops.nhwc_to_nchw(fine, 3)
            elif ctx.need_dimg and dimg_total is not None:
                fine_hw = ctx.states[i].x8.shape
                fine = torch.zeros((fine_hw[0], fine_hw[1], fine_hw[2], 4), device=dimg_total.device)
                ops.avgpool3s2_bwd(ops.nchw_to_nhwc(dimg_total, 4), fine)
                dimg_total = ops.nhwc_to_nchw(fine, 3)
        dx = None
        if ctx.need_dimg:
            dx = torch.zeros(ctx.in_shape, device=gouts[0].device if gouts[0] is not None else None, dtype=torch.float32)
            if dimg_total is not None:
                dx[:, 4:7] = dimg_total
        ctx.states = None
        if not ctx.param_grads:
            return (None, dx) + (None,) * len(ctx.params)
        if red is not None:
            return (None, dx) + red.finish(ctx.params, G.get)
        return (None, dx) + tuple(G.get(p) for p in ctx.params)


def discriminator_forward_autograd(netD, x_nchw):
    params = [p for p in netD.parameters()]
    flat = _DiscriminatorFn.apply(netD, x_nchw, *params)
    children = [D for _, D in netD.named_children()]
    per = children[0].n_layers + 1
    get_feats = not netD.opt.no_ganFeat_loss
    result = []
    for i in range(len(children)):
        outs = list(flat[i * per:(i + 1) * per])
        result.append(outs if get_feats else [outs[-1]])
    return result
