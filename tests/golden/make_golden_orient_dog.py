"""Golden fixture of the reference's DoG orientation loss, generated on the CPU from the LIVE reference:

    python tests/golden/make_golden_orient_dog.py [out.npz]

The unmodified `models.networks.loss.L1OLoss` with orient_filter 'dog' runs its own `forward` in fp32 with two shims that
touch no arithmetic: `Tensor.cuda` returns the tensor itself while the loss runs (DoG_fn and calOrientationDoG move their
parameters with .cuda()), and `1 - <bool tensor>` (loss.py:343) is evaluated as `~<bool tensor>`, the complement the uint8 mask
of the torch the reference was written for gave.  For each case of tests/oracle_orient_dog.py the orientation loss, the
confidence loss and d(10 * ORIENT + 100 * CONFIDENCE)/d(image) are stored in tests/golden/golden_orient_dog.npz.

Every case but 'tie' and 'no_hair' must have a unique maximiser of r * hair, the runner-up below M (1 - 1e-4), so that the
kernels' fp32 responses pick the same pixel; 'tie' has two bit-identical maxima (the same image and hair in both slots).
"""
import contextlib
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
from make_golden_hair_avg_lab import bool_complement  # noqa: E402


@contextlib.contextmanager
def cuda_is_identity():
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = orig


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_orient_dog.npz"))
    import oracle_orient_dog as od
    from michigan_b200.networks.loss import dog_bank
    warnings.filterwarnings("ignore")
    ref_shims.import_reference()
    loss_mod = __import__("models.networks.loss", fromlist=["L1OLoss"])
    bank = dog_bank("cpu")
    res = {}
    for name, (img, label, sem, use_ig) in od.cases().items():
        top = od.top_products(img, sem, bank)
        if name in od.NON_TIE:
            assert top[1] < top[0] * (1 - 1e-4), (name, top)
        elif name == "tie":
            assert top[0] == top[1] and top[2] < top[0] * (1 - 1e-4), (name, top)
        crit = loss_mod.L1OLoss(SimpleNamespace(orient_filter="dog", use_ig=use_ig))
        x = img.clone().requires_grad_()
        with cuda_is_identity(), bool_complement():
            lo, lc = crit(x, label, sem)
        (lo * 10.0 + lc * 100.0).backward()
        xo = img.clone().requires_grad_()
        oo, oc = od.orient_loss_dog(xo, label, sem, use_ig, bank)
        (oo * 10.0 + oc * 100.0).backward()
        if name == "no_hair":
            assert torch.isnan(lo) and torch.isnan(lc) and torch.isnan(x.grad).all()
        else:
            rel = float((xo.grad - x.grad).norm() / x.grad.norm())
            print("%-10s ORIENT %.6f (oracle %.6f)  CONFIDENCE %.6f (oracle %.6f)  grad rel L2 %.2e"
                  % (name, float(lo), float(oo), float(lc), float(oc), rel))
            assert abs(float(oo) - float(lo)) <= 1e-6 * abs(float(lo)) and abs(float(oc) - float(lc)) <= 1e-6 * abs(float(lc))
            assert rel <= 1e-5
        res[name + "_lo"] = np.float64(float(lo))
        res[name + "_lc"] = np.float64(float(lc))
        res[name + "_g"] = x.grad.numpy()
    np.savez_compressed(out, **res)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
