"""Golden fixture of the reference's --remove_background VGG, content and style losses, generated on the CPU from the LIVE
reference:

    python tests/golden/make_golden_remove_background.py [out.npz]

The unmodified `models.networks.loss.VGGLoss` and `StyleContentLoss` with remove_background=True, with the shims of
make_golden_style_content.py, which touch no arithmetic: `torchvision.models.vgg19` returns `vgg19(weights=None)` loaded with
the seeded stand-in weights of michigan_b200.synth (nothing is downloaded), and `.cuda()` is a no-op while the losses are
constructed.  VGGLoss is called as pix2pix_model.py:303-307 does (label = the tag's hair), StyleContentLoss as 309-315
(style_label = the reference image's hair, content_label = the tag's).

Inputs: N = 2 at 64x64, ref != tag, for each case of tests/test_oracle_remove_background.py `_inputs` (different tag and
reference hair masks, an image without tag hair, an image without reference hair, all hair).  The oracle
(tests/oracle_remove_background.py) must agree at fp32 noise level (losses 1e-6 relative, d fake 1e-5 relative L2); then each
loss and d(loss)/d(fake) is stored in tests/golden/golden_remove_background.npz.  The VGG weights are regenerated from the seed.
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
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_remove_background.npz"))
    import torchvision
    from michigan_b200.synth import vgg19_state_dict
    from test_oracle_remove_background import CASES, _inputs, _rel, oracle_terms
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
        opt = SimpleNamespace(remove_background=True)
        vgg = loss_mod.VGGLoss(opt)
        sc = loss_mod.StyleContentLoss(opt)
    finally:
        torchvision.models.vgg19 = real_vgg19
        torch.nn.Module.cuda = cuda
    arrays = {"vgg_seed": np.int64(VGG_SEED)}
    for case in CASES:
        fake, ref, tag, lab_ref, lab_tag = _inputs(case)
        assert not torch.equal(ref, tag)
        reference = {
            "vgg": lambda x: vgg(x, tag, lab_tag),
            "content": lambda x: sc(x, ref, tag, lab_ref, lab_tag)[0],
            "style": lambda x: sc(x, ref, tag, lab_ref, lab_tag)[1],
        }
        oracle = oracle_terms(sd, fake, ref, tag, lab_ref, lab_tag)
        for name in reference:
            lr, gr = _loss_and_grad(reference[name], fake)
            lo, go = _loss_and_grad(oracle[name], fake)
            rel = _rel(go, gr)
            print("%-12s %-8s reference %.8f oracle %.8f  grad rel L2 %.2e" % (case, name, lr, lo, rel))
            assert abs(lo - lr) <= 1e-6 * abs(lr), (case, name)
            assert rel <= 1e-5, (case, name)
            arrays["%s/%s_loss" % (case, name)] = np.float64(lr)
            arrays["%s/%s_grad" % (case, name)] = gr.numpy()
    np.savez_compressed(out, **arrays)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
