"""DANet (ResNet-101 v1c, dilated-8, position + channel attention) training-step benchmark on one GPU: 8 x 769^2 crops,
19 classes (Cityscapes), ProbOhemCrossEntropy2d(thresh 0.7, min_kept = B·H·W/16) on each of the three heads, SGD.

    python tools/bench_danet.py [--batch 8] [--size 769] [--steps 20] [--warmup 5] [--ref-steps 10] [--no-ref]
                                [--attn-iters 20] [--dump-outputs DIR]

Prints one JSON line with
  * the graph-replayed libtsb step (engine.graph.GraphedTrainStep): img/s and ms/step from CUDA events, launches per
    step and peak memory;
  * the same step for the oracle (tests/danet_oracle.py, which materialises the [N, N] and [C, C] attention matrices)
    on cuDNN, strict fp32 and bf16 autocast + channels_last; an out-of-memory arm is reported as such;
  * tsb_attention_fwd / tsb_attention_bwd alone at (B 8, N 9409, d_k 64, d_v 512) (the 769² crop at output stride 8):
    CUDA-event time over many launches and TFLOP/s of the GEMM work the kernels execute, recomputations included
    (forward: S per value slice and P·V, 2·B·N²·(2·64 + 512); backward: S and P·dO per slice in the dV pass, S, dP and
    dS·Q in the dK pass, S, dP and dS·K in the dQ pass, 2·B·N²·(2·(64 + 256) + 2·(64 + 512 + 64)));
  * torch.nn.functional.scaled_dot_product_attention on the same tensors, bf16, as a comparison arm only, with the
    backend it ran on (the first of flash, efficient, cudnn, math that accepts the shape) or the reason none did;
  * ops.ChannelAttentionFn forward + backward alone on 8 x 512 x 97 x 97;
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

from bench_x39 import dump_outputs, gpu_info, time_events  # noqa: E402

BN = torch.nn.BatchNorm2d
SEED = 12345
NUM_CLASSES, IGNORE = 19, 255
DK, DV = 64, 512


def synth_batch(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, h, w, generator=g)
    y = torch.randint(0, NUM_CLASSES, (n, h, w), generator=g, dtype=torch.int64)
    y[:, : h // 10] = IGNORE
    return x, y


def _criterion(n, h, w):
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    return ProbOhemCrossEntropy2d(IGNORE, thresh=0.7, min_kept=n * h * w // 16)


def _model(criterion):
    from torchseg_b200.networks import DANet
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(SEED)
    m = DANet(NUM_CLASSES, criterion, norm_layer=BN)
    init_weight(m.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    with torch.no_grad():   # trained gammas are non-zero; at zero the attention would receive no gradient
        m.head.sa.gamma.fill_(0.5)
        m.head.sc.gamma.fill_(0.25)
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
    import danet_oracle as tr
    from oracle.torch_ref import ohem_ce, resnet_v1c_d8
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
                blocks = resnet_v1c_d8(x, sd, "backbone", (3, 4, 23, 3), 1e-5, 0.1, True, stats)
                heads = tr.danet_head(blocks[-1], sd, "head", 1e-5, 0.1, True, stats)
            up = lambda t: F.interpolate(t.float(), size=(h, w), mode="bilinear", align_corners=True)
            loss = sum(ohem_ce(up(lo), y, IGNORE, 0.7, min_kept) for lo in heads)
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


SDPA_BACKENDS = ("FLASH_ATTENTION", "EFFICIENT_ATTENTION", "CUDNN_ATTENTION", "MATH")


def attention_arm(dev, iters, shapes=((8, 9409),)):
    """tsb_attention_{fwd,bwd} alone at (d_k, d_v) = (64, 512), scale 1 (DANet's position attention), and SDPA (bf16,
    one head) on the same tensors for comparison"""
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from torchseg_b200 import ops
    rows = []
    for B, N in shapes:
        g = torch.Generator(device=dev).manual_seed(1)
        q, k = ((torch.randn(B, N, DK, device=dev, generator=g) * 0.35).to(torch.bfloat16) for _ in range(2))
        v, do = (torch.randn(B, N, DV, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
        o, dv = torch.empty_like(v), torch.empty_like(v)
        dq, dk = torch.empty_like(q), torch.empty_like(q)
        lse = torch.empty(B, N, device=dev)
        delta = torch.empty(B, N, device=dev)
        st = ops.stream()
        calls = {
            "fwd": lambda: ops.call("tsb_attention_fwd", q.data_ptr(), DK, k.data_ptr(), DK, v.data_ptr(), DV,
                                    o.data_ptr(), DV, lse.data_ptr(), B, N, DK, DV, 1.0, st),
            "bwd": lambda: ops.call("tsb_attention_bwd", q.data_ptr(), DK, k.data_ptr(), DK, v.data_ptr(), DV,
                                    o.data_ptr(), DV, do.data_ptr(), DV, lse.data_ptr(), delta.data_ptr(),
                                    dq.data_ptr(), DK, dk.data_ptr(), DK, dv.data_ptr(), DV, 0, B, N, DK, DV, 1.0, st),
        }
        unit = 2.0 * B * N * N
        flop = {"fwd": unit * (2 * DK + DV), "bwd": unit * (2 * (DK + DV // 2) + 2 * (DK + DV + DK))}
        for kind, fn in calls.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ms, _ = time_events(fn, iters)
            rows.append(dict(impl="libtsb", kind=kind, B=B, N=N, d_k=DK, d_v=DV, ms=round(ms, 3),
                             tflop=round(flop[kind] / 1e12, 3), tflops=round(flop[kind] / (ms / 1e3) / 1e12, 1)))
        q4, k4 = (t.view(B, 1, N, DK).detach().requires_grad_(True) for t in (q, k))
        v4 = v.view(B, 1, N, DV).detach().requires_grad_(True)
        do4 = do.view(B, 1, N, DV)
        reasons = {}
        for name in SDPA_BACKENDS:
            try:
                with sdpa_kernel([getattr(SDPBackend, name)]):
                    fwd = lambda: F.scaled_dot_product_attention(q4, k4, v4, scale=1.0)

                    def fwd_bwd():
                        return torch.autograd.grad(fwd(), (q4, k4, v4), do4)

                    for _ in range(3):
                        fwd_bwd()
                    torch.cuda.synchronize()
                    ms_f, _ = time_events(lambda: fwd().detach(), iters)
                    ms_fb, _ = time_events(fwd_bwd, iters)
                rows.append(dict(impl="sdpa", backend=name.lower(), kind="fwd", B=B, N=N, d_k=DK, d_v=DV,
                                 ms=round(ms_f, 3)))
                rows.append(dict(impl="sdpa", backend=name.lower(), kind="fwd+bwd", B=B, N=N, d_k=DK, d_v=DV,
                                 ms=round(ms_fb, 3)))
                break
            except Exception as e:  # noqa: BLE001 — a comparison arm: report, do not hide
                reasons[name.lower()] = str(e).split("\n")[0][:160]
                torch.cuda.empty_cache()
        else:
            rows.append(dict(impl="sdpa", B=B, N=N, d_k=DK, d_v=DV, error="no backend accepted the shape",
                             reasons=reasons))
        if reasons and rows[-1].get("impl") == "sdpa" and "error" not in rows[-1]:
            rows[-1]["rejected_by"] = reasons
        del q, k, v, do, o, dq, dk, dv, q4, k4, v4
        torch.cuda.empty_cache()
    return rows


def cam_arm(dev, iters, B=8, C=512, h=97, w=97):
    """ops.ChannelAttentionFn forward + backward alone (E, soft-max, A·X and their gradients)"""
    from torchseg_b200 import ops
    g = torch.Generator(device=dev).manual_seed(2)
    x = ops.to_nhwc(torch.relu(torch.randn(B, C, h, w, device=dev, generator=g))).requires_grad_(True)
    dy = ops.to_nhwc(torch.randn(B, C, h, w, device=dev, generator=g))

    def fwd_bwd():
        return torch.autograd.grad(ops.ChannelAttentionFn.apply(x), (x,), dy)

    for _ in range(3):
        fwd_bwd()
    torch.cuda.synchronize()
    ms, _ = time_events(fwd_bwd, iters)
    with torch.no_grad():
        ms_f, _ = time_events(lambda: ops.ChannelAttentionFn.apply(x), iters)
    return dict(B=B, C=C, h=h, w=w, fwd_ms=round(ms_f, 3), fwd_bwd_ms=round(ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=769)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=10)
    ap.add_argument("--ref-warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true", help="skip the oracle / cuDNN arms")
    ap.add_argument("--attn-iters", type=int, default=20)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_danet measures the GPU step and needs a CUDA device")
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = dict(metric="danet_r101_train_step", gpu=gpu_info(), size=args.size)
    prod, model, loss = product_arm(dev, args.batch, args.size, args.size, args.steps, args.warmup)
    line["libtsb_graph"] = prod
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, loss, model)
    del model
    torch.cuda.empty_cache()
    line["attention"] = attention_arm(dev, args.attn_iters)
    line["cam"] = cam_arm(dev, args.attn_iters)
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
