"""Evaluator cost per frame, host path against device path, on seeded synthetic frames and labels (no dataset).

  host:   Evaluator.sliding_eval (cv2 / numpy around the network) + metric.hist_info
  device: Evaluator.sliding_eval_device (tsb_eval_* kernels)    + metric.hist_info_torch (n_cl² counts copied back)

The two arms alternate frame by frame in one process, with the same network, frames and labels; every frame's
predictions and confusion matrices must be identical across the arms (asserted). Per workload one JSON line: ms per
frame per arm, the network forward's ms per frame (CUDA events around every val_func call) and its share, the card name
and power limit read in the same run (nvidia-smi, read-only query).

Workloads:
  r18      BiSeNet-R18 eval network (folded BN), 1024x2048 frames, crop 1024, stride 5/6, scale 1, no flip
  r18_ms   the same network and frames, scales 0.5 .. 1.75 with flip
  psp      PSPNet-R101 (150 classes), 512x683 frames, crop 480, stride 2/3, scale 1

Usage: python tools/bench_eval.py [--frames 3] [--workloads r18,r18_ms,psp]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
WORKLOADS = {
    "r18": dict(net="r18", classes=19, hw=(1024, 2048), crop=1024, stride=5 / 6.0, scales=[1.0], flip=False),
    "r18_ms": dict(net="r18", classes=19, hw=(1024, 2048), crop=1024, stride=5 / 6.0,
                   scales=[0.5, 0.75, 1.0, 1.25, 1.5, 1.75], flip=True),
    "psp": dict(net="psp", classes=150, hw=(512, 683), crop=480, stride=2 / 3.0, scales=[1.0], flip=False),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return dict(name=name, power_limit=power)
    except Exception as e:                                  # noqa: BLE001 — the number is still reported
        return dict(name=torch.cuda.get_device_name(0), power_limit="unknown (%s)" % type(e).__name__)


class TimedNet(object):
    """val_func protocol (eval / to / __call__) around a network; CUDA events bracket every forward"""

    def __init__(self, net):
        self.net, self.events = net, []

    def eval(self):
        self.net.eval()
        return self

    def to(self, *a):
        return self

    def __call__(self, x):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        y = self.net(x)
        e1.record()
        self.events.append((e0, e1))
        return y

    def take_ms(self):
        torch.cuda.synchronize()
        ms = sum(a.elapsed_time(b) for a, b in self.events)
        self.events = []
        return ms


def network(kind, classes, dev):
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet, PSPNet
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(12345)
    BN = torch.nn.BatchNorm2d
    if kind == "r18":
        net = BiSeNet(classes, False, None, None, BN)
        init_weight(net.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    else:
        net = PSPNet(classes, torch.nn.CrossEntropyLoss(ignore_index=-1))
    net.to(dev)
    torchseg_b200.prepare_model(net)
    net.eval()
    return net


def run(name, cfg, frames, dev):
    from torchseg_b200.engine.evaluator import Evaluator
    from torchseg_b200.seg_opr.metric import hist_info, hist_info_torch
    net = TimedNet(network(cfg["net"], cfg["classes"], dev))
    ev = Evaluator(dataset=None, class_num=cfg["classes"], image_mean=MEAN, image_std=STD, network=None,
                   multi_scales=cfg["scales"], is_flip=cfg["flip"], devices=[0])
    ev.val_func = net
    rng = np.random.default_rng(7)
    H, W = cfg["hw"]
    n_cl = cfg["classes"]

    def host(img, gt):
        p = ev.sliding_eval(img, cfg["crop"], cfg["stride"], dev)
        return p, hist_info(n_cl, p, gt)[0]

    def device(img, gt):
        p = ev.sliding_eval_device(img, cfg["crop"], cfg["stride"], dev)
        conf = hist_info_torch(n_cl, p, torch.from_numpy(gt).to(dev))[0].cpu().numpy()
        return p, conf

    times = {"host": [], "device": []}
    fwd = {"host": [], "device": []}
    for f in range(frames + 1):                               # frame 0 warms both arms up
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        gt = rng.integers(0, n_cl + 1, (H, W))
        gt[gt == n_cl] = 255
        out = {}
        for arm, fn in (("host", host), ("device", device)) if f % 2 == 0 else (("device", device), ("host", host)):
            torch.cuda.synchronize()
            net.take_ms()
            t0 = time.perf_counter()
            out[arm] = fn(img, gt)
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            fms = net.take_ms()
            if f > 0:
                times[arm].append(dt)
                fwd[arm].append(fms)
        p_dev = out["device"][0].cpu().numpy()
        assert np.array_equal(p_dev, out["host"][0]), "%s frame %d: predictions differ" % (name, f)
        assert np.array_equal(out["device"][1], out["host"][1]), "%s frame %d: confusion matrices differ" % (name, f)
    res = {a: dict(ms_per_frame=float(np.mean(times[a])), ms_per_frame_runs=[round(t, 2) for t in times[a]],
                   forward_ms_per_frame=float(np.mean(fwd[a])), forward_share=float(np.sum(fwd[a]) / np.sum(times[a])))
           for a in times}
    return dict(workload=name, config=dict(cfg, hw=list(cfg["hw"])), frames=frames, host=res["host"], device=res["device"],
                speedup=res["host"]["ms_per_frame"] / res["device"]["ms_per_frame"], identical=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--workloads", default="r18,r18_ms,psp")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval needs cuda:0"
    from torchseg_b200 import build
    build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    gpu = card()
    for name in args.workloads.split(","):
        line = run(name, WORKLOADS[name], args.frames, dev)
        line["gpu"] = gpu
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
