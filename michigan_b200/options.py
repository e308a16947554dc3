"""Default option namespace for the hot path: the subset of the reference's argparse options
(options/base_options.py:22-131, options/train_options.py:12-78) that the generator, discriminator
and losses read, at the README train/inference flag values (README.md:51-60).  When the reference's
own option parser is available (drop-in use) its namespace is used instead; this exists so that the
modules, tests and bench can be constructed stand-alone."""
from types import SimpleNamespace


def make_opt(is_train=True, **overrides):
    o = SimpleNamespace(
        # base options
        name="MichiGAN", gpu_ids=[0], model="pix2pix", norm_G="spectralspadesyncbatch3x3", norm_D="spectralinstance",
        norm_E="spectralinstance", weight_norm_G=False, weight_norm_g=0, batchSize=8, load_size=512, crop_size=512,
        aspect_ratio=1.0, label_nc=2, contain_dontcare_label=False, output_nc=3, orient_nc=2, netG="spadeb", ngf=64,
        init_type="xavier", init_variance=0.02, z_dim=256, use_ig=False, num_upsampling_layers="more",
        use_instance_feat=False, feat_num=3, use_encoder=True, Image_encoder_mode="partialconv",
        ref_global_pool=False, norm_ref_encode="instance", use_blender=False, no_instance=True, use_vae=False, noise_background=True,
        random_expand_mask=True, random_expand_th=0.05, bf_direct_add=False, random_noise_background=False,
        no_orientation=False, add_feat_zeros=False, add_th=64, clip_th=300, use_clip=False, orient_random_disturb=False,
        expand_mask_be=True, expand_th=5, semantic_nc=2, inpaint_mode="ref", only_blend=False, unpairTrain=False,
        curr_step=1, remove_background=False,
        # not a reference option: with remove_background, also mask the VGG, content and style losses (networks.loss.
        # masked_vgg_losses; install() sets it on the reference's own options)
        mask_vgg_losses=False,
        # train options
        ndf=64, netD="multiscale", netD_subarch="n_layer", num_D=2, n_layers_D=4, lambda_feat=1.0, no_gan_loss=False,
        no_ganFeat_loss=False, gan_mode="hinge", no_TTUR=False, lr=0.0002, beta1=0.5, beta2=0.999, wide_edge=2.0,
        # loss switches: the stand-alone model implements hinge GAN + GAN_Feat (SURVEY.md §8d flag set)
        no_vgg_loss=True, no_style_loss=True, no_content_loss=True, no_background_loss=True, no_rgb_loss=True, no_lab_loss=True,
        no_orient_loss=True, no_confidence_loss=True, orient_filter="gabor", lambda_orient=10.0, lambda_confidence=100.0,
        lambda_vgg=1.0, lambda_kld=0.05, lambda_lab=1.0, balance_Lab=False, lambda_content=1.0, lambda_style=1.0, lambda_background=1.0, lambda_rgb=1.0,
        isTrain=is_train,
    )
    for k, v in overrides.items():
        setattr(o, k, v)
    return o
