"""Golden fixture of the reference's VGG perceptual loss and Lab colour loss, generated on the CPU from the LIVE reference:

    python tests/golden/make_golden_vgg_lab.py [out.npz]

VGG: the unmodified `models.networks.loss.VGGLoss` (remove_background False) with two shims that touch no arithmetic:
`torchvision.models.vgg19` returns `vgg19(weights=None)` loaded with the seeded stand-in weights of michigan_b200.synth (nothing
is downloaded; `pretrained=True` never reaches torchvision), and `.cuda()` is a no-op while the loss is constructed.
Lab: the reference's `LabColorLoss.RGB2Lab` (the float-mask formulation, loss.py:414-437, which runs on modern torch) and
`nn.L1Loss` on channels 1: - the same function as its `forward`, whose masked indexing (loss.py:443,474) fails on torch >= 1.2.

The oracle (tests/oracle_vgg_lab.py) must agree at fp32 noise level; then the two losses and d(loss)/d(fake) at N = 2, 64x64
(the inputs of tests/test_oracle_vgg_lab.py) are stored in tests/golden/golden_vgg_lab.npz.  The VGG weights are regenerated
from the seed, not stored.
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


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_vgg_lab.npz"))
    import torchvision
    import oracle_vgg_lab as ovl
    from michigan_b200.synth import vgg19_state_dict
    from test_oracle_vgg_lab import _inputs
    fake, real = _inputs()
    sd = vgg19_state_dict(VGG_SEED)
    warnings.filterwarnings("ignore")
    ref_shims.import_reference()
    os.chdir(ref_shims.REF)
    loss_mod = __import__("models.networks.loss", fromlist=["VGGLoss"])

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
        crit = loss_mod.VGGLoss(SimpleNamespace(remove_background=False))
    finally:
        torchvision.models.vgg19 = real_vgg19
        torch.nn.Module.cuda = cuda
    x = fake.clone().requires_grad_()
    vgg_loss = crit(x, real)
    vgg_loss.backward()
    vgg_grad = x.grad.clone()

    lab = loss_mod.LabColorLoss(SimpleNamespace(balance_Lab=False))
    x = fake.clone().requires_grad_()
    lab_loss = torch.nn.L1Loss()(lab.RGB2Lab((x + 1) / 2.0)[:, 1:], lab.RGB2Lab((real + 1) / 2.0)[:, 1:].detach())
    lab_loss.backward()
    lab_grad = x.grad.clone()

    # the oracle at fp32 noise level
    xo = fake.clone().requires_grad_()
    lo = ovl.vgg_loss(xo, real, sd)
    lo.backward()
    print("VGG loss reference %.8f oracle %.8f  grad rel L2 %.2e" % (float(vgg_loss), float(lo),
                                                                     float((xo.grad - vgg_grad).norm() / vgg_grad.norm())))
    assert abs(float(lo) - float(vgg_loss)) <= 1e-6 * abs(float(vgg_loss))
    assert float((xo.grad - vgg_grad).norm() / vgg_grad.norm()) <= 1e-5
    xo = fake.clone().requires_grad_()
    lo = ovl.lab_loss(xo, real)
    lo.backward()
    print("Lab loss reference %.8f oracle %.8f  grad rel L2 %.2e" % (float(lab_loss), float(lo),
                                                                     float((xo.grad - lab_grad).norm() / lab_grad.norm())))
    assert abs(float(lo) - float(lab_loss)) <= 1e-6 * abs(float(lab_loss))
    assert float((xo.grad - lab_grad).norm() / lab_grad.norm()) <= 1e-6

    np.savez_compressed(out, vgg_seed=np.int64(VGG_SEED), vgg_loss=np.float64(float(vgg_loss)), vgg_grad=vgg_grad.numpy(),
                        lab_loss=np.float64(float(lab_loss)), lab_grad=lab_grad.numpy())
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
