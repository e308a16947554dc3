"""michigan_b200 — an H100-native (sm_90a) implementation of MichiGAN's data-parallel hot path:
the SPADE-conditioned generator (`--netG spadeb`), the multiscale PatchGAN discriminator and
synchronized batch-norm, behind the reference's operator surface and checkpoint layout.

    python -m michigan_b200.build          # nvcc -> michigan_b200/lib/libmichigan_sm90.so (C ABI)
    michigan_b200.install(reference_root)  # plug the networks into the reference's train.py/inference.py
    python -m michigan_b200.launch <reference_root> train.py <flags>   # the same, as a launcher (torchrun for N GPUs)
"""
__version__ = "0.1.0"


def install(reference_root=None, compat=True):
    from .install import install as _install
    return _install(reference_root, compat)
