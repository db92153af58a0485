"""Regenerate tests/golden/live_reference.npz from the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden.py

Stores what the live-reference tests of tests/test_cpu_oracle.py compare against, so that they run without the
reference: OHEM kept sets / losses / sampled gradients, BiSeNet-R18 loss and gradient norms / samples, state_dict keys,
metric outputs, Evaluator outputs (score maps sampled) and DFN block outputs. Everything is seeded.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from golden_cases import bisenet_case, ohem_case  # noqa: E402
from golden_cases import EVAL_KW, OHEM_SAMPLE, eval_image, eval_net, metric_inputs  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference.npz")


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    g = {}
    # OHEM: kept set, loss and a seeded sample of the gradient per (regime, seed)
    lo = rl.load_loss_opr()
    for regime in ["A", "B", "C", "D"]:
        for seed in (1, 2, 3):
            logits, labels, min_kept = ohem_case(regime, seed=seed, H=32, W=40)
            crit = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
            x = logits.clone().requires_grad_(True)
            loss = crit(x, labels)
            loss.backward()
            k = "ohem_%s%d_" % (regime, seed)
            g[k + "kept"] = (x.grad.abs().sum(dim=1) > 0).reshape(-1).numpy()
            g[k + "loss"] = np.float64(float(loss))
            idx = np.random.default_rng(seed).choice(x.grad.numel(), OHEM_SAMPLE, replace=False)
            g[k + "grad_idx"] = idx.astype(np.int32)
            g[k + "grad"] = x.grad.reshape(-1).numpy()[idx]
    # BiSeNet-R18 step: loss bits and every parameter gradient (norm + sample)
    net = rl.load_network('bisenet/cityscapes.bisenet.R18')
    x, y, min_kept, seed = bisenet_case(N=2, HW=64, seed=5)
    torch.manual_seed(seed)
    crit = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    m = net.BiSeNet(19, True, crit, None, torch.nn.BatchNorm2d)
    m.train()
    loss = m(x, y)
    loss.backward()
    g["bisenet_loss"] = np.float32(float(loss))
    # per parameter: gradient norm and a seeded sample of entries (the CPU's conv summation order is not part of the
    # reference, so the test compares with a tolerance rather than bit for bit)
    grads = {}
    for i, (n, p) in enumerate(m.named_parameters()):
        flat = p.grad.reshape(-1).double().numpy()
        idx = np.random.default_rng(i).choice(flat.size, min(flat.size, 64), replace=False)
        grads[n] = [float(np.linalg.norm(flat)), idx.tolist(), flat[idx].tolist()]
    g["bisenet_grads"] = json.dumps(grads)
    # state_dict keys and shapes
    sd = net.BiSeNet(19, True, None, None, torch.nn.BatchNorm2d).state_dict()
    g["bisenet_keys"] = json.dumps([[k, list(v.shape)] for k, v in sd.items()])
    # metric.py
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_metric", os.path.join(rl.REF, "furnace", "seg_opr", "metric.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    n_cl, pred, gt, pr, lab = metric_inputs()
    h, l, c = ref.hist_info(n_cl, pred, gt)
    g["metric_hist"], g["metric_labeled"], g["metric_correct"] = h, np.int64(l), np.int64(c)
    for i, a in enumerate(ref.compute_score(h, c, l)):
        g["metric_score_%d" % i] = np.asarray(a, dtype=np.float64)
    i2, u2 = ref.intersectionAndUnion(pr, lab, 150)
    g["metric_inter"], g["metric_union"] = i2, u2
    for i, a in enumerate(ref.meanIoU(np.stack([i2, i2], 1), np.stack([u2, u2], 1))):
        g["metric_miou_%d" % i] = np.asarray(a, dtype=np.float64)
    g["metric_pixacc"] = np.asarray(ref.pixelAccuracy(pr, lab), dtype=np.float64)
    g["metric_mpa"] = np.float64(ref.mean_pixel_accuracy([3, 4], [5, 6]))
    g["metric_acc"] = np.float64(ref.accuracy(pr, lab)[0])
    # Evaluator on the CPU with a small deterministic network
    ref_mod = rl.load_evaluator()
    torch.Tensor.cuda = lambda self, *a, **k: self
    net_e = eval_net()

    class RefWrap(object):       # the reference calls .eval() / .to(get_device()) (-1 on the CPU) on its val_func
        def eval(self):
            net_e.eval()

        def to(self, *a):
            return self

        def __call__(self, x_):
            return net_e(x_)

    class _DS(object):
        def get_length(self):
            return 0
    ev = ref_mod.Evaluator(**dict(EVAL_KW, dataset=_DS()))
    ev.val_func = RefWrap()
    img = eval_image()
    g["eval_sliding"] = ev.sliding_eval(img, 96, 2 / 3.0, None).astype(np.uint8)
    s = ev.scale_process(img, (150, 210), 96, 2 / 3.0, None)
    g["eval_scale_absmax"] = np.float64(np.abs(s).max())
    sidx = np.random.default_rng(9).choice(s.size, 20000, replace=False)
    g["eval_scale_idx"] = sidx.astype(np.int32)
    g["eval_scale"] = s.reshape(-1)[sidx].astype(np.float32)
    g["eval_small"] = ev.sliding_eval(img[:80, :70], 96, 2 / 3.0, None).astype(np.uint8)
    g["eval_whole"] = ev.whole_eval(img, (75, 105), (160, 224), None).astype(np.uint8)
    g["eval_grey"] = ev.whole_eval(img[:, :, :1], None, None, None).astype(np.uint8)
    # DFN blocks (fp32, train mode) on seeded inputs and seeded module initialisation
    so = rl.load_seg_oprs()
    torch.manual_seed(3)
    x = torch.randn(2, 16, 9, 11)
    for relu in (True, False):
        for name, mk in (("bnrefine", lambda: so.BNRefine(16, 16, 3, has_relu=relu)),
                         ("refres", lambda: so.RefineResidual(16, 24, 3, has_relu=relu))):
            mod = mk().train()
            g["dfn_%s_%d_sd" % (name, relu)] = json.dumps({k: v.tolist() for k, v in mod.state_dict().items()})
            g["dfn_%s_%d_out" % (name, relu)] = mod(x).detach().numpy()
    mod = so.ChannelAttention(32, 16, 1)
    x2 = torch.randn(2, 16, 9, 11)
    g["dfn_ca_sd"] = json.dumps({k: v.tolist() for k, v in mod.state_dict().items()})
    g["dfn_ca_out"] = mod(x, x2).detach().numpy()
    g["dfn_x"], g["dfn_x2"] = x.numpy(), x2.numpy()
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
