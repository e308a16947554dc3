"""Golden fixture of the reference networks' state-dict layout and seeded initial weights, generated from the LIVE reference:

    python tests/golden/make_golden_layout.py

The unmodified `define_G` / `define_D` (ngf = ndf = 32, 128x128) are built once without a seed (layout: key order, shapes,
dtypes) and `define_G` once more after torch.manual_seed(123) (initial weights).  Each initial tensor is stored as a
fingerprint (float64 sum and sum of squares, and 16 elements at fixed flat positions); tests/test_host_logic.py checks the
host networks against tests/golden/golden_layout.npz without the reference.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_shims  # noqa: E402

ARGS = ["--ngf", "32", "--ndf", "32", "--crop_size", "128", "--load_size", "128"]
INIT_SEED = 123


def fingerprint(t):
    """[sum, sum of squares, 16 elements at flat positions i * numel // 16] in float64."""
    f = t.detach().reshape(-1).double()
    idx = [i * f.numel() // 16 for i in range(16)] if f.numel() else []
    return [float(f.sum()), float((f * f).sum())] + [float(f[i]) for i in idx]


def layout(sd):
    return [[k, list(v.shape), str(v.dtype)] for k, v in sd.items()]


def main():
    ref_shims.patch_training()
    opt = ref_shims.ref_options(True, ARGS)
    nets = ref_shims.import_reference()
    with contextlib.redirect_stdout(io.StringIO()):
        refG, refD = nets.define_G(opt), nets.define_D(opt)
    torch.manual_seed(INIT_SEED)
    with contextlib.redirect_stdout(io.StringIO()):
        initG = nets.define_G(opt)
    init = initG.state_dict()
    # layouts as JSON text ([key, shape, dtype] rows), fingerprints as one float64 row per key in state-dict order
    np.savez_compressed(os.path.join(HERE, "golden_layout.npz"), init_seed=np.int64(INIT_SEED),
                        G=np.array(json.dumps(layout(refG.state_dict()))), D=np.array(json.dumps(layout(refD.state_dict()))),
                        G_init_keys=np.array(json.dumps(list(init.keys()))),
                        G_init=np.array([fingerprint(v) for v in init.values()], dtype=np.float64))
    print("wrote golden_layout.npz: %d G keys, %d D keys" % (len(refG.state_dict()), len(refD.state_dict())))


if __name__ == "__main__":
    main()
