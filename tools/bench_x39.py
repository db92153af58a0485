"""BiSeNet-X39 training-step benchmark on one GPU (the X39 config: 16 x 1024^2 crops, OHEM, SGD).

    python tools/bench_x39.py [--batch 16] [--size 1024] [--steps 20] [--warmup 5] [--ref-steps 10] [--no-ref]
                              [--dw-iters 50] [--dump-outputs DIR]

Prints one JSON line with
  * the graph-replayed libtsb step (engine.graph.GraphedTrainStep): img/s and ms/step from CUDA events;
  * the same step for the oracle (tests/x39_oracle.py: the reference's stock torch.nn lowering) on cuDNN, strict fp32
    and bf16 autocast + channels_last, as bench.py's reference arm does;
  * every depthwise-conv launch shape of the step (fprop, dgrad, wgrad): kernel time from CUDA events over many
    launches, achieved GB/s against the algorithmic bytes (each operand read or written once, computed from the shape),
    and that rate's share of the H100 SXM's 3.35 TB/s;
  * the card name, power limit and max SM clock (nvidia-smi, read-only query) of the run.
--dump-outputs DIR writes the last timed step's loss and a seeded sample of the updated parameters (.npy), so two runs
can be compared bit for bit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the X39 oracle (test infrastructure) for the reference arm

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
NUM_CLASSES, IGNORE = 19, 255
DUMP_PARAM_SAMPLE = 1 << 20


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e)[:200])


def synth_batch(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, h, w, generator=g)
    y = torch.randint(0, NUM_CLASSES, (n, h, w), generator=g, dtype=torch.int64)
    y[:, : h // 10] = IGNORE
    return x, y


def build(dev, n, h, w):
    import torchseg_b200
    from torchseg_b200 import optim
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight, group_weight
    BN = torch.nn.BatchNorm2d
    torch.manual_seed(12345)
    ohem = ProbOhemCrossEntropy2d(ignore_label=IGNORE, thresh=0.7, min_kept=n * h * w // 16, use_weight=False)
    model = BiSeNet(NUM_CLASSES, True, torch.nn.CrossEntropyLoss(ignore_index=IGNORE), ohem, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    model.to(dev)
    torchseg_b200.prepare_model(model)
    model.train()
    groups = group_weight([], model.context_path, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return model, optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)


def time_events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, out


def product_arm(dev, n, h, w, steps, warmup):
    from torchseg_b200.engine.graph import GraphedTrainStep
    model, opt = build(dev, n, h, w)
    x, y = synth_batch(n, h, w, 7)
    x, y = x.to(dev), y.to(dev)
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
                final_loss=loss, launches_per_step=step.launches_per_step), model, loss


def reference_arm(dev, n, h, w, steps, warmup, mode, sd0):
    """the oracle step under cuDNN (benchmark on); 'fp32' strict, 'bf16' autocast + channels_last"""
    import torch.nn.functional as F
    import x39_oracle as torch_ref
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
        min_kept, stats = n * h * w // 16, {}

        def one():
            opt.zero_grad()
            if mode == "bf16":
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    lo, _ = torch_ref.bisenet_x39_forward(x, sd, 1e-5, 0.1, True, stats)
                loss = 0
                for l, sc in zip([l.float() for l in lo], (16, 8, 8)):
                    up = F.interpolate(l, scale_factor=sc, mode="bilinear", align_corners=True)
                    loss = loss + torch_ref.ohem_ce(up, y, IGNORE, 0.7, min_kept)
            else:
                loss, _ = torch_ref.bisenet_x39_loss(x, y, sd, min_kept, stats=stats)
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


def dw_shapes(n, size):
    """(C, input H = W, stride, launches per step) of every depthwise conv of the X39 forward"""
    s = size // 4   # stem /2, max-pool /2
    out = []
    for C_in, mid, nblk in ((8, 16, 4), (64, 32, 8), (128, 64, 4)):
        out.append((C_in, s, 2, 2))            # proj and residual_branch.0 of the projecting block
        s = (s - 1) // 2 + 1
        out.append((mid, s, 1, 2 * nblk))      # residual_branch.1 / .2 of every block
        out.append((mid * 4, s, 1, nblk - 1))  # residual_branch.0 of the identity blocks
    return out


def dw_kernel_arm(dev, n, size, iters):
    from torchseg_b200 import ops
    rows = []
    for C, H, st, mult in dw_shapes(n, size):
        P = (H - 1) // st + 1
        cs = (C + 63) // 64 * 64   # the network reads / writes these convs inside 64-padded buffers
        x = torch.randn(n, H, H, cs, device=dev).to(torch.bfloat16)
        dy = torch.randn(n, P, P, cs, device=dev).to(torch.bfloat16)
        y = torch.empty(n, P, P, cs, device=dev, dtype=torch.bfloat16)
        dx = torch.empty(n, H, H, cs, device=dev, dtype=torch.bfloat16)
        w = torch.randn(C, 9, device=dev)
        dw = torch.zeros(C, 9, device=dev)
        s = ops.stream()
        calls = {
            "fprop": lambda: ops.call("tsb_dwconv_fprop", x.data_ptr(), cs, w.data_ptr(), y.data_ptr(), cs, n, H, H, C, st, s),
            "dgrad": lambda: ops.call("tsb_dwconv_dgrad", dy.data_ptr(), cs, w.data_ptr(), dx.data_ptr(), cs, n, H, H, C, st,
                                      0, s),
            "wgrad": lambda: ops.call("tsb_dwconv_wgrad", x.data_ptr(), cs, dy.data_ptr(), cs, dw.data_ptr(), n, H, H, C,
                                      st, *ops.det_ws(), s),
        }
        act_in, act_out = 2.0 * n * H * H * C, 2.0 * n * P * P * C
        nbytes = {"fprop": act_in + act_out + 36 * C, "dgrad": act_in + act_out + 36 * C, "wgrad": act_in + act_out + 72 * C}
        for kind, fn in calls.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ms, _ = time_events(fn, iters)
            gbs = nbytes[kind] / (ms / 1e3) / 1e9
            rows.append(dict(kind=kind, N=n, C=C, H=H, W=H, stride=st, cs=cs, per_step=mult, us=round(ms * 1e3, 2),
                             bytes=int(nbytes[kind]), GBps=round(gbs, 1), hbm_share=round(gbs * 1e9 / HBM_BYTES_PER_S, 3)))
        del x, dy, y, dx
    total_us = sum(r["us"] * r["per_step"] for r in rows)
    return rows, total_us


def dump_outputs(out_dir, loss, model):
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    params = torch.cat([p.detach().float().reshape(-1) for p in model.parameters()]).cpu().numpy()
    idx = np.sort(np.random.default_rng(0).choice(params.size, min(DUMP_PARAM_SAMPLE, params.size), replace=False))
    np.save(os.path.join(out_dir, "loss.npy"), np.array([loss], dtype=np.float32))
    np.save(os.path.join(out_dir, "params_sample.npy"), params[idx].astype(np.float32))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=10)
    ap.add_argument("--ref-warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true", help="skip the oracle / cuDNN arms")
    ap.add_argument("--dw-iters", type=int, default=50)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_x39 measures the GPU step and needs a CUDA device")
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = dict(metric="bisenet_x39_train_step", gpu=gpu_info(), size=args.size)
    prod, model, loss = product_arm(dev, args.batch, args.size, args.size, args.steps, args.warmup)
    line["libtsb_graph"] = prod
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, loss, model)
    del model
    torch.cuda.empty_cache()
    rows, total_us = dw_kernel_arm(dev, args.batch, args.size, args.dw_iters)
    line["dwconv"] = dict(launches=rows, weighted_us_per_step=round(total_us, 1))
    if not args.no_ref:
        sd0 = _initial_state()
        for mode in ("fp32", "bf16"):
            try:
                line["reference_%s" % mode] = reference_arm(dev, args.batch, args.size, args.size, args.ref_steps,
                                                            args.ref_warmup, mode, sd0)
            except torch.cuda.OutOfMemoryError as e:
                line["reference_%s" % mode] = dict(error="out of memory: %s" % str(e).split("\n")[0][:160])
                torch.cuda.empty_cache()
    print(json.dumps(line))


def _initial_state():
    """the product arm's initial weights (same seed, same init), on the host"""
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    from torchseg_b200.utils.init_func import init_weight
    BN = torch.nn.BatchNorm2d
    torch.manual_seed(12345)
    m = BiSeNet(NUM_CLASSES, True, None, None, None, BN)
    init_weight(m.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


if __name__ == "__main__":
    main()
