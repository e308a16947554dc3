"""Shims that let the UNMODIFIED reference scripts run in an offline / modern-PyTorch environment.  None of them
touches arithmetic on the hot path:

  1. `matplotlib` / `dominate` are imported by reference modules but unused on the train / inference path
     (generator.py:9, normalization.py:13, util/html.py:7-8): stubbed only when they are not installed;
  2. `torch.optim.Adam(betas=(0, 0.9))` with the int 0 (pix2pix_model.py:141-145) is rejected by torch >= 2.x:
     betas are coerced to float;
  3. `networks.StyleContentLoss` is constructed unconditionally (pix2pix_model.py:47) and needs the VGG19 weights
     (loss.py:659, architecture.py:163): when BOTH --no_style_loss and --no_content_loss are given its result is
     discarded (pix2pix_model.py:310-319), so whatever class is bound (install() binds michigan_b200's) is replaced by a
     zero stub in that case only.
"""
import importlib
import sys
import types


def stub_optional_imports():
    for name, attrs in (("matplotlib", ()), ("matplotlib.pyplot", ()), ("dominate", ("document",)), ("dominate.tags", ())):
        if name in sys.modules:
            continue
        try:
            importlib.import_module(name)
        except Exception:
            m = types.ModuleType(name)
            for a in attrs:
                setattr(m, a, object)
            sys.modules[name] = m
            if "." in name:
                parent, child = name.rsplit(".", 1)
                setattr(sys.modules[parent], child, m)


def patch_adam_betas():
    import torch
    if getattr(torch.optim.Adam, "_mg_float_betas", False):
        return
    orig = torch.optim.Adam.__init__

    def init(self, params, lr=1e-3, betas=(0.9, 0.999), **kw):
        orig(self, params, lr=lr, betas=(float(betas[0]), float(betas[1])), **kw)

    torch.optim.Adam.__init__ = init
    torch.optim.Adam._mg_float_betas = True


def patch_style_content_loss(networks_pkg):
    import torch
    orig = networks_pkg.StyleContentLoss
    if getattr(orig, "_mg_lazy", False):
        return

    class StyleContentLoss(torch.nn.Module):
        _mg_lazy = True

        def __init__(self, opt=None, *a, **k):
            super().__init__()
            unused = opt is not None and getattr(opt, "no_style_loss", False) and getattr(opt, "no_content_loss", False)
            self.impl = None if unused else orig(opt, *a, **k)

        def forward(self, *a, **k):
            if self.impl is None:
                return 0, 0
            return self.impl(*a, **k)

    networks_pkg.StyleContentLoss = StyleContentLoss
