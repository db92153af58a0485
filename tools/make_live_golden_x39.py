"""Write tests/golden/live_reference_x39.npz from the unmodified reference BiSeNet-X39 network.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_x39.py

Stores what tests/test_cpu_x39.py compares against, so that it runs without the reference: the seeded training loss,
every parameter gradient's norm and 64 seeded entries, and the state_dict keys and shapes.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from golden_cases import bisenet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_x39.npz")


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    g = {}
    lo = rl.load_loss_opr()
    net = rl.load_network('bisenet/cityscapes.bisenet.X39')
    x, y, min_kept, seed = bisenet_case(N=2, HW=64, seed=5)
    torch.manual_seed(seed)
    crit = torch.nn.CrossEntropyLoss(reduction='mean', ignore_index=255)
    ohem = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    m = net.BiSeNet(19, True, crit, ohem, None, torch.nn.BatchNorm2d)
    m.train()
    loss = m(x, y)
    loss.backward()
    g["x39_loss"] = np.float32(float(loss))
    grads = {}
    for i, (n, p) in enumerate(m.named_parameters()):
        flat = p.grad.reshape(-1).double().numpy()
        idx = np.random.default_rng(i).choice(flat.size, min(flat.size, 64), replace=False)
        grads[n] = [float(np.linalg.norm(flat)), idx.tolist(), flat[idx].tolist()]
    g["x39_grads"] = json.dumps(grads)
    sd = net.BiSeNet(19, True, None, None, None, torch.nn.BatchNorm2d).state_dict()
    g["x39_keys"] = json.dumps([[k, list(v.shape)] for k, v in sd.items()])
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
