"""Write tests/golden/live_reference_bisenet_lines.npz from the unmodified reference BiSeNet networks R18.speed,
X39.speed and R101.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_bisenet_lines.py

Stores what tests/test_cpu_bisenet_lines.py compares against, so that it runs without the reference: for each line the
seeded training loss, every parameter gradient's norm and 64 seeded entries, and the state_dict keys and shapes of the
training and of the eval network. The .speed lines run at N=2, 64x128 with labels at 1/8 (8x16) and the .speed
min_kept; R101 at N=2, 64x64 with full-resolution labels.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bisenet_lines_cases import bisenet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_bisenet_lines.npz")

# line → (reference directory, bisenet_case arguments, takes ohem_criterion)
LINES = {
    "r18_speed": ("bisenet/cityscapes.bisenet.R18.speed", dict(N=2, H=64, W=128, gt_down=8, seed=21), True),
    "x39_speed": ("bisenet/cityscapes.bisenet.X39.speed", dict(N=2, H=64, W=128, gt_down=8, seed=22), True),
    "r101": ("bisenet/cityscapes.bisenet.R101", dict(N=2, H=64, W=64, seed=23), False),
}


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    g = {}
    lo = rl.load_loss_opr()
    for name, (rel, case, two_crit) in LINES.items():
        net = rl.load_network(rel)
        x, y, min_kept, seed = bisenet_case(**case)
        torch.manual_seed(seed)
        ohem = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
        if two_crit:
            crit = torch.nn.CrossEntropyLoss(reduction='mean', ignore_index=255)
            m = net.BiSeNet(19, True, crit, ohem, None, torch.nn.BatchNorm2d)
        else:
            m = net.BiSeNet(19, True, ohem, None, torch.nn.BatchNorm2d)
        m.train()
        loss = m(x, y)
        loss.backward()
        g[name + "_loss"] = np.float32(float(loss))
        grads = {}
        for i, (n, p) in enumerate(m.named_parameters()):
            flat = p.grad.reshape(-1).double().numpy()
            idx = np.random.default_rng(i).choice(flat.size, min(flat.size, 64), replace=False)
            grads[n] = [float(np.linalg.norm(flat)), idx.tolist(), flat[idx].tolist()]
        g[name + "_grads"] = json.dumps(grads)
        for mode, training in (("train", True), ("eval", False)):
            args = (19, training, None, None, None, torch.nn.BatchNorm2d) if two_crit else \
                (19, training, None, None, torch.nn.BatchNorm2d)
            sd = net.BiSeNet(*args).state_dict()
            g["%s_%s_keys" % (name, mode)] = json.dumps([[k, list(v.shape)] for k, v in sd.items()])
        print(name, float(loss))
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
