"""Operator layer of the hot path — the classes the reference looks up by name in
`models.networks.{generator,discriminator,normalization,architecture,encoder,sync_batchnorm}`
(models/networks/__init__.py:16-85), re-implemented on hand-written sm_90a kernels."""
import torch

from .base_network import BaseNetwork
from .normalization import SPADE, get_nonspade_norm_layer
from .architecture import SPADEResnetBlock, VGG19
from . import loss
from .loss import GANLoss, GANFeatLoss, VGGLoss, LabColorLoss, StyleContentLoss, RGBBackgroundL1Loss, HairAvgLabLoss, KLDLoss
from .encoder import ImageEncoder, ImageEncoder2, ImageEncoder3, BackgroundEncode2, PartialConv2d, ConvBlock, ConvEncoder
from .generator import SPADEBGenerator
from .discriminator import MultiscaleDiscriminator, NLayerDiscriminator
from .inpaint import InpaintGenerator
from . import sync_batchnorm
from .sync_batchnorm import SynchronizedBatchNorm2d, DataParallelWithCallback

_GENERATORS = {"spadeb": SPADEBGenerator, "inpaint": InpaintGenerator}
_DISCRIMINATORS = {"multiscale": MultiscaleDiscriminator, "nlayer": NLayerDiscriminator, "n_layer": NLayerDiscriminator}
_ENCODERS = {"conv": ConvEncoder}


def find_network_using_name(target_network_name, filename):
    """networks/__init__.py:16-24: `<name><filename>` looked up case-insensitively."""
    table = {"generator": _GENERATORS, "discriminator": _DISCRIMINATORS, "encoder": _ENCODERS}.get(filename)
    if table is None or target_network_name.lower() not in table:
        raise ValueError("In %s.py, there should be a class name that matches %s in lowercase (michigan_b200 "
                         "implements netG=spadeb, netD=multiscale)" % (filename, target_network_name + filename))
    return table[target_network_name.lower()]


def modify_commandline_options(parser, is_train):
    opt, _ = parser.parse_known_args()
    parser = find_network_using_name(opt.netG, "generator").modify_commandline_options(parser, is_train)
    if is_train:
        parser = find_network_using_name(opt.netD, "discriminator").modify_commandline_options(parser, is_train)
    return parser


def create_network(cls, opt):
    """networks/__init__.py:41-48; unlike the reference a GPU is mandatory (no CPU path exists)."""
    net = cls(opt)
    net.print_network()
    if len(opt.gpu_ids) > 0:
        assert torch.cuda.is_available()
        net.cuda()
    net.init_weights(opt.init_type, opt.init_variance)
    return net


def define_G(opt):
    return create_network(find_network_using_name(opt.netG, "generator"), opt)


def define_IG(opt):
    """networks/__init__.py:70-72 (`--netIG inpaint`): the frozen orientation-inpainting net of --use_ig."""
    return create_network(find_network_using_name(getattr(opt, "netIG", "inpaint"), "generator"), opt)


def define_D(opt):
    return create_network(find_network_using_name(opt.netD, "discriminator"), opt)


def define_E(opt):
    """networks/__init__.py:65-68: the --use_vae image encoder (there is one encoder type, 'conv')."""
    return create_network(find_network_using_name("conv", "encoder"), opt)
