"""Golden fixture of the reference's Gabor orientation loss, generated on a GPU machine from the LIVE reference (its
`L1OLoss` hard-codes .cuda()):

    python tests/golden/make_golden_orient.py [out.npz]

The unmodified `models.networks.loss.L1OLoss` (orient_filter gabor) runs in fp32 (TF32 convolutions off: the arg-max over
32 close filter responses must not depend on operand rounding) on the fixed inputs of tests/test_gpu_orient.py.  Its
orientation loss, confidence loss and d(10 * lo + 100 * lc)/d(image) are stored in tests/golden/golden_orient.npz, which
tests/test_gpu_orient.py compares the oracle against without the reference.
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
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_orient.npz"))
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from test_gpu_orient import _inputs
    from michigan_b200 import compat
    img, orient, sem = _inputs()
    sys.path.insert(0, ref_shims.REF)
    compat.stub_optional_imports()
    warnings.filterwarnings("ignore")
    os.chdir(ref_shims.REF)
    from models.networks.loss import L1OLoss
    crit = L1OLoss(SimpleNamespace(orient_filter="gabor", use_ig=False))
    x = img.cuda().requires_grad_()
    lo, lc = crit(x, orient.cuda(), sem.cuda())
    (lo * 10.0 + lc * 100.0).backward()
    np.savez_compressed(out, lo=lo.detach().cpu().numpy(), lc=lc.detach().cpu().numpy(), g=x.grad.cpu().numpy())
    print("wrote", out, float(lo), float(lc))


if __name__ == "__main__":
    main()
