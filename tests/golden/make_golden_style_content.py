"""Golden fixture of the reference's style, content, background and rgb losses, generated on the CPU from the LIVE reference:

    python tests/golden/make_golden_style_content.py [out.npz]

Style / content: the unmodified `models.networks.loss.StyleContentLoss` (remove_background False), with the shims of
make_golden_vgg_lab.py, which touch no arithmetic: `torchvision.models.vgg19` returns `vgg19(weights=None)` loaded with the
seeded stand-in weights of michigan_b200.synth (nothing is downloaded), and `.cuda()` is a no-op while the loss is constructed.
Background: the unmodified `RGBBackgroundL1Loss`.  rgb: `nn.L1Loss()(fake, tag.detach())`, as pix2pix_model.py:51, 328-333.

Inputs: N = 2 at 64x64 with ref != tag (tests/test_oracle_style_content.py `_inputs`).  The oracle (tests/oracle_style_content.py)
must agree at fp32 noise level (losses 1e-6 relative, d fake 1e-5 relative L2); then each loss and d(loss)/d(fake) is stored in
tests/golden/golden_style_content.npz.  The VGG weights are regenerated from the seed, not stored.
"""
import os
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ref_shims  # noqa: E402

VGG_SEED = 0


def _loss_and_grad(fn, fake):
    x = fake.clone().requires_grad_()
    loss = fn(x)
    loss.backward()
    return float(loss), x.grad.clone()


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_style_content.npz"))
    import torchvision
    import oracle_style_content as osc
    from michigan_b200.synth import vgg19_state_dict
    from test_oracle_style_content import _inputs
    fake, ref, tag, sem = _inputs()
    assert not torch.equal(ref, tag)
    sd = vgg19_state_dict(VGG_SEED)
    warnings.filterwarnings("ignore")
    ref_shims.import_reference()
    os.chdir(ref_shims.REF)
    loss_mod = __import__("models.networks.loss", fromlist=["StyleContentLoss"])

    real_vgg19 = torchvision.models.vgg19

    def seeded_vgg19(*a, **k):
        m = real_vgg19(weights=None)
        missing, _ = m.load_state_dict(sd, strict=False)
        assert all(not n.startswith("features.") for n in missing), missing
        return m

    cuda = torch.nn.Module.cuda
    torchvision.models.vgg19 = seeded_vgg19
    torch.nn.Module.cuda = lambda self, *a, **k: self
    try:
        crit = loss_mod.StyleContentLoss(SimpleNamespace(remove_background=False))
    finally:
        torchvision.models.vgg19 = real_vgg19
        torch.nn.Module.cuda = cuda
    bg = loss_mod.RGBBackgroundL1Loss()
    l1 = torch.nn.L1Loss()
    reference = {
        "content": lambda x: crit(x, ref, tag)[0],
        "style": lambda x: crit(x, ref, tag)[1],
        "background": lambda x: bg(x, sem, tag),
        "rgb": lambda x: l1(x, tag.detach()),
    }
    oracle = {
        "content": lambda x: osc.style_content_loss(x, ref, tag, sd)[0],
        "style": lambda x: osc.style_content_loss(x, ref, tag, sd)[1],
        "background": lambda x: osc.background_loss(x, sem, tag),
        "rgb": lambda x: osc.rgb_loss(x, tag),
    }
    arrays = {"vgg_seed": np.int64(VGG_SEED)}
    for name in reference:
        lr, gr = _loss_and_grad(reference[name], fake)
        lo, go = _loss_and_grad(oracle[name], fake)
        rel = float((go - gr).norm() / gr.norm())
        print("%-10s reference %.8f oracle %.8f  grad rel L2 %.2e" % (name, lr, lo, rel))
        assert abs(lo - lr) <= 1e-6 * abs(lr), name
        assert rel <= 1e-5, name
        arrays[name + "_loss"] = np.float64(lr)
        arrays[name + "_grad"] = gr.numpy()
    np.savez_compressed(out, **arrays)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
