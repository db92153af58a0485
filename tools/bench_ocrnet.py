"""OCRNet (ResNet-101 v1c, dilated-8) training-step benchmark on one GPU: 8 x 769^2 crops, 19 classes (Cityscapes),
ProbOhemCrossEntropy2d(thresh 0.7, min_kept = B·H·W/16), SGD.

    python tools/bench_ocrnet.py [--batch 8] [--size 769] [--steps 20] [--warmup 5] [--ref-steps 10] [--no-ref]
                                 [--op-iters 20] [--dump-outputs DIR]

Prints one JSON line with
  * the graph-replayed libtsb step (engine.graph.GraphedTrainStep): img/s and ms/step from CUDA events, launches per
    step and peak memory;
  * the same step for the oracle (tests/ocrnet_oracle.py) on cuDNN, strict fp32 and bf16 autocast + channels_last;
  * the OCR head's own operations alone at the 769² crop (B 8, a 97 x 97 map, K 19): tsb_cross_attention_fwd / bwd at
    (Nq 9409, Nk 19), and ops.SpatialGatherFn forward and forward + backward (the spatial soft-max and the per-image
    GEMMs), CUDA-event time over many launches;
  * the card name, power limit and max SM clock (nvidia-smi, read-only query) of the run.
--dump-outputs DIR writes the last timed step's loss and a seeded sample of the updated parameters (.npy), so two runs
can be compared bit for bit.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the oracle (test infrastructure) for the reference arm
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_ocnet import IGNORE, NUM_CLASSES, _criterion, synth_batch  # noqa: E402
from bench_x39 import dump_outputs, gpu_info, time_events  # noqa: E402

BN = torch.nn.BatchNorm2d
SEED = 12345
D = 256


def _model(criterion):
    from torchseg_b200.networks import OCRNet
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(SEED)
    m = OCRNet(NUM_CLASSES, criterion, norm_layer=BN)
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
    import ocrnet_oracle as tr
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
                lo, dsn = tr.ocrnet_logits(x, sd, 1e-5, 0.1, True, stats)
            up = lambda t: F.interpolate(t.float(), size=(h, w), mode="bilinear", align_corners=True)
            loss = (ohem_ce(up(lo), y, IGNORE, 0.7, min_kept) + 0.4 * ohem_ce(up(dsn), y, IGNORE, 0.7, min_kept))
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


def op_arm(dev, iters, B=8, h=97, w=97, K=NUM_CLASSES):
    """the cross attention at (B, Nq = h·w, Nk = K) and the gather at (B, 512, h, w, K) alone"""
    from torchseg_b200 import ops
    rows = []
    Nq = h * w
    g = torch.Generator(device=dev).manual_seed(1)
    q, do = (torch.randn(B, Nq, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(B, K, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    o, dq = torch.empty_like(q), torch.empty_like(q)
    dk, dv = torch.empty_like(k), torch.empty_like(v)
    lse, delta = torch.empty(B, Nq, device=dev), torch.empty(B, Nq, device=dev)
    st = ops.stream()
    s = D ** -0.5
    calls = {
        "cross_attention_fwd": lambda: ops.call(
            "tsb_cross_attention_fwd", q.data_ptr(), D, k.data_ptr(), D, v.data_ptr(), D, o.data_ptr(), D,
            lse.data_ptr(), B, Nq, K, D, D, s, st),
        "cross_attention_bwd": lambda: ops.call(
            "tsb_cross_attention_bwd", q.data_ptr(), D, k.data_ptr(), D, v.data_ptr(), D, o.data_ptr(), D,
            do.data_ptr(), D, lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), D, dk.data_ptr(), D, dv.data_ptr(), D,
            B, Nq, K, D, D, s, st),
    }
    f = ops.to_nhwc(torch.randn(B, 512, h, w, device=dev, generator=g)).requires_grad_(True)
    lcs = (K + 31) // 32 * 32
    logits = ops.nhwc_zeros(B, K, h, w, dtype=torch.float32, device=dev, cs=lcs)
    with torch.no_grad():
        logits.copy_(torch.randn(B, K, h, w, device=dev, generator=g) * 3)
    logits.requires_grad_(True)
    dctx = ops.to_nhwc(torch.randn(B, 512, K, 1, device=dev, generator=g))

    def gather_fwd():
        with torch.no_grad():
            return ops.SpatialGatherFn.apply(f, logits, K)

    def gather_fwd_bwd():
        return torch.autograd.grad(ops.SpatialGatherFn.apply(f, logits, K), (f, logits), dctx)

    calls["gather_fwd"] = gather_fwd
    calls["gather_fwd+bwd"] = gather_fwd_bwd
    for kind, fn in calls.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms, _ = time_events(fn, iters)
        rows.append(dict(kind=kind, B=B, Nq=Nq, Nk=K, ms=round(ms, 3)))
    del q, do, k, v, o, dq, dk, dv, f, logits
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
    ap.add_argument("--op-iters", type=int, default=20)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ocrnet measures the GPU step and needs a CUDA device")
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = dict(metric="ocrnet_r101_train_step", gpu=gpu_info(), size=args.size)
    prod, model, loss = product_arm(dev, args.batch, args.size, args.size, args.steps, args.warmup)
    line["libtsb_graph"] = prod
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, loss, model)
    del model
    torch.cuda.empty_cache()
    line["ops"] = op_arm(dev, args.op_iters)
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
