"""Golden fixture of the reference's count-balanced Lab losses (--balance_Lab), generated on the CPU from the LIVE reference:

    python tests/golden/make_golden_balance_lab.py [out.npz]

The unmodified `models.networks.loss.LabColorLoss` and `HairAvgLabLoss` run their own `forward` with balance_Lab True, with two
shims that touch no arithmetic:
  1. each instance's `FloatTensor`, hard-coded as torch.cuda.FloatTensor (loss.py:407, 538), is torch.FloatTensor, the CPU
     fp32 constructor of the same table;
  2. while the losses run, `1 - <bool tensor>` is `~<bool tensor>`, what the uint8 masks of the torch the reference was
     written for gave (xyz2lab's `1 - mask`; make_golden_hair_avg_lab.bool_complement).

The count table is synthetic (tests/oracle_balance_lab.count_table, from the seed stored here), written to a temporary file as
--weight_dir, and used with Lab_weight_th 10 and 2.5.  The inputs are tests/oracle_balance_lab.golden_inputs (bins at least
1e-3 from a rounding boundary).  The oracle must agree at fp32 noise level; then the losses and d(loss)/d(fake) of both classes
are stored in tests/golden/golden_balance_lab.npz.
"""
import os
import sys
import tempfile
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


def reference_losses(weight_dir, th):
    """(LabColorLoss, HairAvgLabLoss) of the live reference with balance_Lab, on the CPU (shim 1)."""
    ref_shims.import_reference()
    loss_mod = __import__("models.networks.loss", fromlist=["LabColorLoss"])
    opt = SimpleNamespace(balance_Lab=True, weight_dir=weight_dir, Lab_weight_th=th)
    lab, avg = loss_mod.LabColorLoss(opt), loss_mod.HairAvgLabLoss(opt)
    lab.FloatTensor = avg.FloatTensor = torch.FloatTensor
    return lab, avg


def _grad(fn, fake):
    x = fake.clone().requires_grad_()
    with bool_complement():
        loss = fn(x)
    loss.backward()
    return loss.detach(), x.grad.clone()


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_balance_lab.npz"))
    import oracle_balance_lab as obl
    warnings.filterwarnings("ignore")
    table = obl.count_table(obl.TABLE_SEED)
    res = {"table_seed": np.int64(obl.TABLE_SEED), "thresholds": np.array(obl.THRESHOLDS)}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "ab_count.npy")
        np.save(path, table)
        for th in obl.THRESHOLDS:
            lab, avg = reference_losses(path, th)
            w = obl.weight_map(table, th)
            for name, (fake, real, mf, mr) in obl.golden_inputs().items():
                key = "%s_th%g" % (name, th)
                runs = (("lab", lambda x: lab(x, real, mf), lambda x: obl.lab_color_loss_balanced(x, real, mf, w)),
                        ("avg", lambda x: avg(x, real, mf, mr), lambda x: obl.hair_avg_lab_loss_balanced(x, real, mf, mr, w)))
                for cls, ref_fn, orc_fn in runs:
                    loss, grad = _grad(ref_fn, fake)
                    lo, go = _grad(orc_fn, fake)
                    rel = float((go - grad).norm() / grad.norm())
                    print("%-3s %-16s reference %.8f oracle %.8f  grad rel L2 %.2e" % (cls, key, float(loss), float(lo), rel))
                    assert abs(float(lo) - float(loss)) <= 1e-6 * abs(float(loss))
                    assert rel <= 1e-5
                    res["%s_%s_loss" % (cls, key)] = np.float64(float(loss))
                    res["%s_%s_grad" % (cls, key)] = grad.numpy()
    np.savez_compressed(out, **res)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
