"""DenseASPP (ResNet-101 v1c, dilated-8) training-step benchmark on one GPU: 8 x 769^2 crops, 19 classes (Cityscapes),
ProbOhemCrossEntropy2d(thresh 0.7, min_kept = B·H·W/16), SGD.

    python tools/bench_denseaspp.py [--batch 8] [--size 769] [--steps 20] [--warmup 5] [--ref-steps 10] [--no-ref]
                                    [--kernel-iters 20] [--dump-outputs DIR]

Prints one JSON line with
  * the graph-replayed libtsb step (engine.graph.GraphedTrainStep): img/s and ms/step from CUDA events, launches per
    step and peak memory;
  * the same step for the oracle (tests/denseaspp_oracle.py, which writes the normalised copy of every block's input)
    on cuDNN, strict fp32 and bf16 autocast + channels_last; an out-of-memory arm is reported as such;
  * the pre-activation 1x1 kernels alone at the four shapes of blocks 1-4 (75 272 pixels = 8 x 97², C = 2176 ... 2560,
    K = 512), CUDA-event time over many launches: tsb_conv1x1_bnrelu_fprop (statistics epilogue) against tsb_bn_apply +
    tsb_conv2d_fprop, and tsb_conv1x1_bnrelu_wgrad against tsb_bn_apply + tsb_conv2d_wgrad, with TFLOP/s of the GEMM
    (2·pixels·C·K per call); the head's 1x1 forward is 888 GFLOP and its 3x3 forward 444 GFLOP per step;
  * the card name, power limit and max SM clock (nvidia-smi, read-only query) of the run.
--dump-outputs DIR writes the last timed step's loss and a seeded sample of the updated parameters (.npy), so two runs
can be compared bit for bit.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the oracle (test infrastructure) for the reference arm
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_ocnet import synth_batch, _criterion  # noqa: E402
from bench_x39 import dump_outputs, gpu_info, time_events  # noqa: E402

BN = torch.nn.BatchNorm2d
SEED = 12345
NUM_CLASSES, IGNORE = 19, 255


def _model(criterion):
    from torchseg_b200.networks import DenseASPP
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(SEED)
    m = DenseASPP(NUM_CLASSES, criterion, norm_layer=BN)
    init_weight(m.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    return m


def build(dev, n, h, w):
    import torchseg_b200
    from torchseg_b200 import optim
    from torchseg_b200.utils.init_func import group_weight
    model = _model(_criterion(n, h, w))
    model.to(dev)
    torchseg_b200.prepare_model(model)
    model.train()
    groups = group_weight([], model.backbone, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return model, optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)


def product_arm(dev, n, h, w, steps, warmup):
    from torchseg_b200.engine.graph import GraphedTrainStep
    model, opt = build(dev, n, h, w)
    x, y = synth_batch(n, h, w, 7)
    x, y = x.to(dev), y.to(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    torch.cuda.set_stream(torch.cuda.Stream())
    step = GraphedTrainStep(model, opt, [x, y], warmup=2)
    if step.graph is None:
        raise RuntimeError("CUDA graph capture failed: %s" % step.error)
    for _ in range(warmup):
        step(x, y)
    torch.cuda.synchronize()
    ms, loss = time_events(lambda: step(x, y), steps)
    loss = float(loss.detach())
    torch.cuda.set_stream(torch.cuda.default_stream())
    return dict(value=n / (ms / 1e3), unit="images/sec", ms_per_step=ms, batch=n, steps=steps, warmup=warmup,
                final_loss=loss, launches_per_step=step.launches_per_step,
                peak_memory_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)), model, loss


def reference_arm(dev, n, h, w, steps, warmup, mode, sd0):
    """the oracle step under cuDNN (benchmark on); 'fp32' strict, 'bf16' autocast + channels_last"""
    import torch.nn.functional as F
    import denseaspp_oracle as tr
    from oracle.torch_ref import ohem_ce
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = mode != "fp32"
    try:
        sd, params = {}, []
        for k, v in sd0.items():
            v = v.detach().clone().to(dev)
            if mode == "bf16" and v.dim() == 4:
                v = v.contiguous(memory_format=torch.channels_last)
            if v.is_floating_point() and "running" not in k:
                v.requires_grad_(True)
                params.append(v)
            sd[k] = v
        opt = torch.optim.SGD(params, lr=1e-2, momentum=0.9, weight_decay=5e-4)
        x, y = synth_batch(n, h, w, 7)
        x, y = x.to(dev), y.to(dev)
        if mode == "bf16":
            x = x.contiguous(memory_format=torch.channels_last)
        stats = {}
        min_kept = n * h * w // 16

        def one():
            opt.zero_grad()
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
                lo = tr.denseaspp_logits(x, sd, 1e-5, 0.1, True, stats)
            up = F.interpolate(lo.float(), size=(h, w), mode="bilinear", align_corners=True)
            loss = ohem_ce(up, y, IGNORE, 0.7, min_kept)
            loss.backward()
            opt.step()
            return loss

        for _ in range(warmup):
            one()
        torch.cuda.synchronize()
        ms, loss = time_events(one, steps)
        return dict(value=n / (ms / 1e3), unit="images/sec", ms_per_step=ms, steps=steps, warmup=warmup,
                    final_loss=float(loss.detach()))
    finally:
        torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        torch.cuda.empty_cache()


def kernel_arm(dev, iters, npix=8 * 97 * 97, K=512, widths=(2176, 2304, 2432, 2560)):
    """the fused pre-activation 1x1 fprop / wgrad against tsb_bn_apply + the plain conv, per block shape"""
    from torchseg_b200 import ops
    rows = []
    for C in widths:
        g = torch.Generator(device=dev).manual_seed(C)
        x = ops.to_nhwc(torch.randn(1, C, 1, npix, device=dev, generator=g))
        dy = ops.to_nhwc(torch.randn(1, K, 1, npix, device=dev, generator=g))
        aux = torch.randn(4, C, device=dev, generator=g).contiguous()
        wb = (torch.randn(K, 1, 1, C, device=dev, generator=g) * C ** -0.5).to(torch.bfloat16).contiguous()
        y = ops.nhwc_empty(1, K, 1, npix, device=dev)
        xh = ops.nhwc_empty(1, C, 1, npix, device=dev)
        dw = torch.zeros(K, 1, 1, C, device=dev)
        st = torch.zeros(2, K, device=dev)
        shp = ops.make_shape(1, 1, npix, C, K, 1, 1, 0, 1)
        s = ops.stream()
        ws = ops.det_ws()

        def bn_apply():
            ops.call("tsb_bn_apply", ops.ptr(x), C, ops.ptr(aux[2]), ops.ptr(aux[3]), None, 0, 1, ops.ptr(xh), C, npix, C, s)

        calls = {
            "fprop_fused": lambda: ops.call("tsb_conv1x1_bnrelu_fprop", ctypes.byref(shp), ops.ptr(x), C, ops.ptr(aux[2]),
                                            ops.ptr(aux[3]), ops.ptr(wb), None, 0, ops.ptr(y), 1, K, ops.ptr(st[0]),
                                            ops.ptr(st[1]), *ws, s),
            "fprop_pair": lambda: (bn_apply(), ops.call("tsb_conv2d_fprop", ctypes.byref(shp), ops.ptr(xh), C, ops.ptr(wb),
                                                        None, ops.ptr(y), 1, K, ops.ptr(st[0]), ops.ptr(st[1]), *ws, s)),
            "wgrad_fused": lambda: ops.call("tsb_conv1x1_bnrelu_wgrad", ctypes.byref(shp), ops.ptr(x), C, ops.ptr(aux[2]),
                                            ops.ptr(aux[3]), ops.ptr(dy), K, ops.ptr(dw), *ws, s),
            "wgrad_pair": lambda: (bn_apply(), ops.call("tsb_conv2d_wgrad", ctypes.byref(shp), ops.ptr(xh), C, ops.ptr(dy),
                                                        K, ops.ptr(dw), *ws, s)),
        }
        flop = 2.0 * npix * C * K
        row = dict(C=C, K=K, pixels=npix, gflop=round(flop / 1e9, 1))
        for name, fn in calls.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ms, _ = time_events(fn, iters)
            row[name + "_ms"] = round(ms, 3)
            row[name + "_tflops"] = round(flop / (ms / 1e3) / 1e12, 1)
        rows.append(row)
        del x, dy, xh, y
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=769)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=10)
    ap.add_argument("--ref-warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true", help="skip the oracle / cuDNN arms")
    ap.add_argument("--kernel-iters", type=int, default=20)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_denseaspp measures the GPU step and needs a CUDA device")
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = dict(metric="denseaspp_r101_train_step", gpu=gpu_info(), size=args.size)
    prod, model, loss = product_arm(dev, args.batch, args.size, args.size, args.steps, args.warmup)
    line["libtsb_graph"] = prod
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, loss, model)
    del model
    torch.cuda.empty_cache()
    line["preact_1x1"] = kernel_arm(dev, args.kernel_iters)
    if not args.no_ref:
        sd0 = {k: v.detach().clone() for k, v in _model(None).state_dict().items()}
        for mode in ("fp32", "bf16"):
            try:
                line["reference_%s" % mode] = reference_arm(dev, args.batch, args.size, args.size, args.ref_steps,
                                                            args.ref_warmup, mode, sd0)
            except torch.cuda.OutOfMemoryError as e:
                line["reference_%s" % mode] = dict(error="out of memory: %s" % str(e).split("\n")[0][:160])
                torch.cuda.empty_cache()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
