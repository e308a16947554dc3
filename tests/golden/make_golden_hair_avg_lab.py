"""Golden fixture of the reference's hair-average Lab loss (the unpaired stage's colour term), generated on the CPU from the
LIVE reference:

    python tests/golden/make_golden_hair_avg_lab.py [out.npz]

The unmodified `models.networks.loss.HairAvgLabLoss` (balance_Lab False) runs its own `forward`, with one shim that touches no
arithmetic: its `f()` and `xyz2lab()` index with `1 - mask` on the bool tensor `input > 0.008856` (loss.py:546, 565), which
torch >= 1.2 refuses.  Under the torch the reference was written for, the comparison returned a uint8 mask and `1 - mask` its
complement.  While the loss runs, `1 - <bool tensor>` is therefore evaluated as `~<bool tensor>`, the float-free
equivalent of that complement, so every other line of the class runs as written.

The oracle (tests/oracle_unpaired.py) must agree at fp32 noise level; then the loss and d(loss)/d(fake) of the three cases of
tests/test_oracle_unpaired.py (N = 2, 48x48) are stored in tests/golden/golden_hair_avg_lab.npz.
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


@contextlib.contextmanager
def bool_complement():
    """`1 - mask` on a bool tensor -> `~mask` (what the uint8 masks of torch < 1.2 gave)."""
    orig = torch.Tensor.__rsub__

    def rsub(self, other):
        if self.dtype == torch.bool and isinstance(other, int) and other == 1:
            return ~self
        return orig(self, other)

    torch.Tensor.__rsub__ = rsub
    try:
        yield
    finally:
        torch.Tensor.__rsub__ = orig


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_hair_avg_lab.npz"))
    import oracle_unpaired as ou
    from test_oracle_unpaired import CASES, cases
    warnings.filterwarnings("ignore")
    ref_shims.import_reference()
    loss_mod = __import__("models.networks.loss", fromlist=["HairAvgLabLoss"])
    crit = loss_mod.HairAvgLabLoss(SimpleNamespace(balance_Lab=False))
    res = {}
    for name in CASES:
        fake, real, mf, mr = cases()[name]
        x = fake.clone().requires_grad_()
        with bool_complement():
            loss = crit(x, real, mf, mr)
        loss.backward()
        grad = x.grad.clone()
        xo = fake.clone().requires_grad_()
        lo = ou.hair_avg_lab_loss(xo, real, mf, mr)
        lo.backward()
        rel = float((xo.grad - grad).norm() / grad.norm())
        print("%-15s reference %.8f oracle %.8f  grad rel L2 %.2e" % (name, float(loss), float(lo), rel))
        assert abs(float(lo) - float(loss)) <= 1e-6 * abs(float(loss))
        assert rel <= 1e-5
        res[name + "_loss"] = np.float64(float(loss))
        res[name + "_grad"] = grad.numpy()
    np.savez_compressed(out, **res)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
