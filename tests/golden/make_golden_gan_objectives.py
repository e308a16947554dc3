"""Golden fixture of the reference's adversarial losses, generated on the CPU from the LIVE reference:

    python tests/golden/make_golden_gan_objectives.py [out.npz]

The unmodified `models.networks.loss.GANLoss` (tensor=torch.FloatTensor) and `GANFeatLoss` (gpu_ids=[]) run their own
`__call__` / `forward` on the cases of tests/test_oracle_gan_objectives.py: every gan_mode, non-default target labels, the
wide-edge weight map, and --remove_background with a hair label, a full one and an empty one.  No shim is needed.

The oracle (tests/oracle_gan_objectives.py) must agree at fp32 noise level; then each case's loss and the gradient of the
loss w.r.t. its differentiable inputs (the logits for GANLoss, the intermediate features for GANFeatLoss) are stored in
tests/golden/golden_gan_objectives.npz.
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


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_gan_objectives.npz"))
    import test_oracle_gan_objectives as tg
    warnings.filterwarnings("ignore")
    ref_shims.import_reference()
    loss_mod = __import__("models.networks.loss", fromlist=["GANLoss", "GANFeatLoss"])

    def ref_gan(mode, rl, fl, we, rb):
        return loss_mod.GANLoss(mode, target_real_label=rl, target_fake_label=fl, tensor=torch.FloatTensor,
                                opt=SimpleNamespace(wide_edge=we, remove_background=rb))

    def ref_feat(rb):
        return loss_mod.GANFeatLoss(SimpleNamespace(gpu_ids=[], lambda_feat=tg.LAMBDA_FEAT, remove_background=rb))

    res = {}
    runs = [(name, tg.run_gan, ref_gan, tg.oracle_gan) for name in tg.GAN_CASES]
    runs += [(name, tg.run_feat, ref_feat, tg.oracle_feat) for name in tg.FEAT_CASES]
    for name, run, ref, orc in runs:
        loss, grad = run(name, ref)
        lo, go = run(name, orc)
        err = float((go - grad).abs().max())
        print("%-32s reference %.8f oracle %.8f  grad max err %.2e" % (name, float(loss), float(lo), err))
        assert abs(float(lo) - float(loss)) <= 1e-6 * abs(float(loss)) + 1e-12
        assert err <= 1e-6 * float(grad.abs().max()) + 1e-12
        res[name + "_loss"] = np.float64(float(loss))
        res[name + "_grad"] = grad.numpy()
    np.savez_compressed(out, **res)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
