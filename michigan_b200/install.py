"""Drop the sm_90a operator classes into an (unmodified) MichiGAN checkout.

The reference resolves networks by *name* at run time: `find_class_in_module(name + 'generator',
'models.networks.generator')` scans the module's __dict__ (util/util.py:180-192,
models/networks/__init__.py:16-24), and the trainer imports `DataParallelWithCallback` from
`models.networks.sync_batchnorm` (trainers/pix2pix_trainer.py:6).  Rebinding those names before the
options are parsed is therefore enough for `train.py` / `inference.py` to run on the CUDA kernels
with no source change (see INTEGRATION.md for the launcher).
"""
import importlib
import os
import sys


def install(reference_root=None, compat=True):
    """Import the reference's `models.networks` package and rebind the hot-path classes; then adapt the runtime
    around them to one process per GPU (`_patch_runtime`).  compat=True also applies the offline / modern-PyTorch
    shims of michigan_b200.compat (none touches hot-path arithmetic)."""
    if reference_root:
        reference_root = os.path.abspath(reference_root)
        if reference_root not in sys.path:
            sys.path.insert(0, reference_root)
    if compat:
        from . import compat as _compat
        _compat.stub_optional_imports()
        _compat.patch_adam_betas()
    from . import networks as mine
    gen = importlib.import_module("models.networks.generator")
    dis = importlib.import_module("models.networks.discriminator")
    nrm = importlib.import_module("models.networks.normalization")
    arc = importlib.import_module("models.networks.architecture")
    enc = importlib.import_module("models.networks.encoder")
    sbn = importlib.import_module("models.networks.sync_batchnorm")
    base = importlib.import_module("models.networks.base_network")
    pkg = importlib.import_module("models.networks")
    # the factory asserts issubclass(cls, <reference BaseNetwork>) (models/networks/__init__.py:21-22):
    # derive the installed network classes from both bases (same names, lookup is by module attribute)
    def both(cls):
        if issubclass(cls, base.BaseNetwork):
            return cls
        return type(cls.__name__, (cls, base.BaseNetwork), {"__doc__": cls.__doc__, "__module__": cls.__module__})

    G = both(mine.SPADEBGenerator)
    MSD = both(mine.MultiscaleDiscriminator)
    NLD = both(mine.NLayerDiscriminator)
    gen.SPADEBGenerator = G
    gen.SPADEResnetBlock = mine.SPADEResnetBlock
    gen.ImageEncoder3 = mine.ImageEncoder3
    gen.ImageEncoder = mine.ImageEncoder
    gen.ImageEncoder2 = mine.ImageEncoder2
    gen.BackgroundEncode2 = mine.BackgroundEncode2
    dis.MultiscaleDiscriminator = MSD
    dis.NLayerDiscriminator = NLD
    nrm.SPADE = mine.SPADE
    nrm.SynchronizedBatchNorm2d = mine.SynchronizedBatchNorm2d
    arc.SPADEResnetBlock = mine.SPADEResnetBlock
    arc.SPADE = mine.SPADE
    enc.ImageEncoder3 = mine.ImageEncoder3
    enc.ImageEncoder = mine.ImageEncoder
    enc.ImageEncoder2 = mine.ImageEncoder2
    enc.BackgroundEncode2 = mine.BackgroundEncode2
    # --use_vae: define_E finds 'convencoder' in models.networks.encoder (networks/__init__.py:65-68)
    enc.ConvEncoder = both(mine.ConvEncoder)
    for name in ("SynchronizedBatchNorm1d", "SynchronizedBatchNorm2d", "SynchronizedBatchNorm3d", "DataParallelWithCallback",
                 "patch_replication_callback", "convert_model", "patch_sync_batchnorm"):
        setattr(sbn, name, getattr(mine.sync_batchnorm, name))
    pkg.SPADEBGenerator, pkg.MultiscaleDiscriminator, pkg.NLayerDiscriminator = G, MSD, NLD
    # the GAN and GAN feature-matching losses (pix2pix_model.py:36-39, networks.GANLoss, networks.GANFeatLoss), the perceptual,
    # style / content, background and Lab colour losses (pix2pix_model.py:41-53 look them up as networks.VGGLoss,
    # networks.StyleContentLoss, networks.RGBBackgroundL1Loss, networks.LabColorLoss) and the hair-average Lab loss of the
    # unpaired stage (pix2pix_model.py:55-56, networks.HairAvgLabLoss), and the KL divergence of --use_vae (pix2pix_model.py:42-43,
    # networks.KLDLoss).  The rgb term is a bare nn.L1Loss (pix2pix_model.py:51)
    # and stays torch's: torch.nn is not patched.
    los = importlib.import_module("models.networks.loss")
    for name in ("GANLoss", "GANFeatLoss", "VGGLoss", "StyleContentLoss", "RGBBackgroundL1Loss", "LabColorLoss", "HairAvgLabLoss",
                 "KLDLoss"):
        setattr(los, name, getattr(mine.loss, name))
        setattr(pkg, name, getattr(mine.loss, name))
    if getattr(gen, "InpaintGenerator", None) is not None:
        IG = both(mine.InpaintGenerator)
        gen.InpaintGenerator = IG
        pkg.InpaintGenerator = IG
    if compat:
        _compat.patch_style_content_loss(pkg)
    _patch_runtime()
    return mine


def _patch_runtime():
    """What changes around the networks under one process per GPU (nothing in the reference's files is edited):

      * `util.save_network` (util/util.py:195-200) -> michigan_b200.checkpoint.save_network: rank 0 only, atomic rename,
        barrier, no round trip of the whole network through the CPU;
      * `Pix2PixModel.__init__`: under --remove_background it sets opt.mask_vgg_losses, so the installed VGGLoss and
        StyleContentLoss compute the reference's hair-masked terms (networks.loss.masked_vgg_losses);
      * `Pix2PixModel.compute_generator_loss` (pix2pix_model.py:257-365): the discriminators' parameters (netD, and netD2
        of --unpairTrain, which judges the generator in the unpaired stage, pix2pix_model.py:568-572) do not require grad
        while the GENERATOR's loss is back-propagated - the reference computes those gradients and throws them away
        (optimizer_D.zero_grad() / optimizer_D2.zero_grad() run before they could be used, pix2pix_trainer.py:61-77), here
        they are not computed (and not all-reduced) at all.  Gradient averaging itself needs no hook: it happens inside
        backward() (networks/sync_batchnorm.GradReducer, one per network), so the unchanged Pix2PixTrainer is data-parallel
        as is."""
    from . import checkpoint
    util_mod = importlib.import_module("util.util")
    util_mod.save_network = checkpoint.save_network
    pm = importlib.import_module("models.pix2pix_model")
    cls = pm.Pix2PixModel
    if not getattr(cls, "_mg_patched", False):
        orig = cls.compute_generator_loss

        def compute_generator_loss(self, *a, **k):
            nets = [n for n in (getattr(self, "netD", None), getattr(self, "netD2", None)) if n is not None]
            flags = [(p, p.requires_grad) for n in nets for p in n.parameters()]
            for p, _ in flags:
                p.requires_grad_(False)
            try:
                return orig(self, *a, **k)
            finally:
                for p, r in flags:
                    p.requires_grad_(r)

        cls.compute_generator_loss = compute_generator_loss
        orig_init = cls.__init__

        def __init__(self, opt, *a, **k):
            # the reference's --remove_background masks its VGG, content and style losses too (loss.py:187-207, 634-711): opt
            # into the masked terms of networks.loss.VGGLoss / StyleContentLoss, which refuse the flag alone
            if getattr(opt, "remove_background", False):
                opt.mask_vgg_losses = True
            orig_init(self, opt, *a, **k)

        cls.__init__ = __init__
        cls._mg_patched = True
