#!/usr/bin/env python
"""bench.py — images/sec of the BiSeNet-R18 training step (1024x1024, 19 classes, bf16, batch 16/GPU, OHEM).

    python bench.py --gpus N --steps K --warmup W            # H100-native path (libtsb)
    python bench.py ... --dump-outputs DIR                   # also write the last timed step's results as .npy
    python bench.py --impl reference --gpus N --steps K ...  # reference CPU arm (oracle port on host cores)

One "step" = zero_grad → forward (3 OHEM losses) → backward → gradient all-reduce (N>1) → fused SGD step, i.e.
TorchSeg model/bisenet/cityscapes.bisenet.R18/train.py:116-142 on synthetic data (SURVEY.md §8d).
Prints ONE JSON line (rank 0). See the task contract for the keys.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

H = W = 1024
NUM_CLASSES = 19
IGNORE = 255
BATCH_PER_GPU = 16
STEP_GFLOP_PER_IMG = 338.1   # BASELINE.md §2: 3 x 116.00 - 2 x 4.933 (conv FLOPs, fprop+dgrad+wgrad)
METRIC = "images/sec training step (1024x1024, 19-class)"
MODEL = "bisenet"            # --model pspnet: secondary line for BASELINE configs[2] (PSPNet-R101_v1c d8, ADE shape)
WORKLOAD = "BiSeNet-R18 train step, 1024x1024, 19-class, OHEM (BASELINE configs[1])"
CPU_SAMPLE_BATCH = 2         # the CPU arms time batch 2 @ 1024x1024 per step (one shape for cpu_baseline and --impl reference)


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm_gbs=d["hbm_gbs"], tflops=d.get("bf16_tflops_sustained", d["bf16_tflops"]), src="measured (sustained)")
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s
    return dict(hbm_gbs=3350.0, tflops=989.0, src="H100 SXM data sheet")


# ------------------------------------------------------------------------------------------------ data
def synth_batch(n, h, w, seed, device="cpu", pin=False):
    g = torch.Generator().manual_seed(seed)
    imgs = torch.randn(n, 3, h, w, generator=g)
    labels = torch.randint(0, NUM_CLASSES, (n, h, w), generator=g, dtype=torch.int64)
    labels[:, : h // 10, :] = IGNORE  # deterministic ~10 % ignore band
    batch = [imgs, labels]
    if MODEL == "dfn":   # border labels {0,1,255} (dfn dataloader.py:15-29 produces them with Canny + dilate)
        edge = (torch.rand(n, h, w, generator=g) < 0.1).to(torch.int64)
        edge[:, : h // 10, :] = IGNORE
        batch.append(edge)
    if pin and torch.cuda.is_available():
        batch = [t.pin_memory() for t in batch]
    return tuple(t.to(device) for t in batch)


# ------------------------------------------------------------------------------------------------ clocks
class ClockSampler(object):
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index, self.rows, self.stop = index, [], False
        self.t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self.stop:
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5).stdout
                self.rows.append([c.strip() for c in out.strip().split(",")])
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.2)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *a):
        self.stop = True
        self.t.join(timeout=6)

    def summary(self):
        sm = sorted(int(r[0]) for r in self.rows if len(r) >= 6 and r[0].isdigit())
        mx = [int(r[1]) for r in self.rows if len(r) >= 6 and r[1].isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) >= 6 and r[2 + i].lower().startswith("active") for r in self.rows)]
        return dict(sm_mhz=sm[len(sm) // 2] if sm else None, sm_max_mhz=max(mx) if mx else None, reasons=reasons,
                    samples=len(self.rows))


# ------------------------------------------------------------------------------------------------ model
def build_b200(device, world):
    import torchseg_b200
    from torchseg_b200 import optim
    from torchseg_b200.apex.parallel import DistributedDataParallel, SyncBatchNorm
    from torchseg_b200.engine.lr_policy import PolyLR
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight, group_weight
    norm = SyncBatchNorm if world > 1 else torch.nn.BatchNorm2d
    if MODEL in ("pspnet", "psanet"):
        # model/{pspnet,psanet}/ade.*.R101_v1c/train.py:47-90: CE(ignore -1), backbone lr, business layers 10x lr
        from torchseg_b200.networks import PSPNet, PSANet
        if MODEL == "psanet":
            PSPNet = PSANet
        torch.manual_seed(304)
        model = PSPNet(NUM_CLASSES, torch.nn.CrossEntropyLoss(reduction='mean', ignore_index=-1), None, norm)
        for mod in model.modules():
            if isinstance(mod, torch.nn.Dropout2d):
                mod.p = 0.1
        init_weight(model.business_layer, torch.nn.init.kaiming_normal_, norm, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
        model.to(device)
        torchseg_b200.prepare_model(model)
        base_lr = 1e-2
        groups = group_weight([], model.backbone, norm, base_lr)
        for m in model.business_layer:
            groups = group_weight(groups, m, norm, base_lr * 10)
        opt = optim.SGD(groups, lr=base_lr, momentum=0.9, weight_decay=1e-4)
        lr_policy = PolyLR(base_lr, 0.9, 120 * 1000)
        ddp = DistributedDataParallel(model) if world > 1 else None
        model.train()
        return model, ddp, opt, lr_policy
    if MODEL == "dfn":
        # model/dfn/cityscapes.dfn.R101_v1c/train.py:47-80: CE(ignore 255) + 0.1 * focal, backbone lr, business 10x lr
        from torchseg_b200.networks import DFN
        from torchseg_b200.seg_opr.loss_opr import SigmoidFocalLoss
        torch.manual_seed(12345)
        model = DFN(NUM_CLASSES, torch.nn.CrossEntropyLoss(reduction='mean', ignore_index=255),
                    SigmoidFocalLoss(ignore_label=255, gamma=2.0, alpha=0.25), 0.1, None, norm)
        init_weight(model.business_layer, torch.nn.init.kaiming_normal_, norm, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
        model.to(device)
        torchseg_b200.prepare_model(model)
        base_lr = 7e-4
        groups = group_weight([], model.backbone, norm, base_lr)
        for m in model.business_layer:
            groups = group_weight(groups, m, norm, base_lr * 10)
        opt = optim.SGD(groups, lr=base_lr, momentum=0.9, weight_decay=1e-4)
        lr_policy = PolyLR(base_lr, 0.9, 80 * 1000)
        ddp = DistributedDataParallel(model) if world > 1 else None
        model.train()
        return model, ddp, opt, lr_policy
    min_kept = BATCH_PER_GPU * H * W // 16  # train.py:48-49
    crit = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    torch.manual_seed(12345)
    model = BiSeNet(NUM_CLASSES, True, crit, None, norm)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, norm, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    model.to(device)
    torchseg_b200.prepare_model(model)
    base_lr = 1e-2
    groups = group_weight([], model.context_path, norm, base_lr)
    for m in (model.spatial_path, model.global_context, model.arms, model.refines, model.heads, model.ffm):
        groups = group_weight(groups, m, norm, base_lr * 10)
    opt = optim.SGD(groups, lr=base_lr, momentum=0.9, weight_decay=5e-4)
    lr_policy = PolyLR(base_lr, 0.9, 80 * 1000)
    ddp = DistributedDataParallel(model) if world > 1 else None
    model.train()
    return model, ddp, opt, lr_policy


def train_step(model, ddp, opt, lr_policy, it, *inputs):
    opt.zero_grad()
    loss = (ddp or model)(*inputs)
    lr = lr_policy.get_lr(it)
    for i, g in enumerate(opt.param_groups):
        g['lr'] = lr if i < 2 else lr * 10  # train.py:136-139
    loss.backward()
    if ddp is not None:
        ddp.finish_reduce()
    opt.step()
    return loss


# ------------------------------------------------------------------------------------------------ CPU arm
def cpu_reference_steps(n, h, w, steps, warmup, threads):
    """The reference algorithm (oracle/torch_ref.py restatement, fp32, NCHW, stock torch.nn lowering) driving the
    same zero_grad → forward(loss) → backward → SGD step sequence on the host CPU."""
    from oracle import torch_ref
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.utils.init_func import init_weight
    torch.set_num_threads(threads)
    torch.manual_seed(12345)
    shell = BiSeNet(NUM_CLASSES, True, None, None, torch.nn.BatchNorm2d)
    init_weight(shell.business_layer, torch.nn.init.kaiming_normal_, torch.nn.BatchNorm2d, 1e-5, 0.1, mode='fan_in',
                nonlinearity='relu')
    sd = {k: v.detach().clone() for k, v in shell.state_dict().items()}
    params = []
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
            params.append(v)
    opt = torch.optim.SGD(params, lr=1e-2, momentum=0.9, weight_decay=5e-4)
    imgs, gts = synth_batch(n, h, w, 7)
    min_kept = n * h * w // 16
    times = []
    for it in range(warmup + steps):
        t0 = time.perf_counter()
        opt.zero_grad()
        loss, _ = torch_ref.bisenet_r18_loss(imgs, gts, sd, min_kept)
        loss.backward()
        opt.step()
        dt = time.perf_counter() - t0
        if it >= warmup:
            times.append(dt)
    return n * len(times) / sum(times), float(loss.detach())


def gpu_reference_steps(device, n, h, w, steps, warmup, mode):
    """SURVEY §8d last row / BASELINE.md §3: the reference step (oracle/torch_ref.py restatement = the reference
    modules' stock torch.nn lowering) on THIS GPU under cuDNN with cudnn.benchmark=True (train.py:35) and
    torch.optim.SGD — the practical "reference GPU path". mode: 'fp32' (strict, TF32 off), 'tf32' (PyTorch's conv
    default) or 'bf16' (torch.autocast + channels_last, the fastest stock-PyTorch configuration). The oracle is the thing
    COMPARED AGAINST here, never part of the product path."""
    from oracle import torch_ref
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.utils.init_func import init_weight
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = mode != "fp32"
    torch.backends.cuda.matmul.allow_tf32 = mode != "fp32"
    try:
        torch.manual_seed(12345)
        shell = BiSeNet(NUM_CLASSES, True, None, None, torch.nn.BatchNorm2d)
        init_weight(shell.business_layer, torch.nn.init.kaiming_normal_, torch.nn.BatchNorm2d, 1e-5, 0.1, mode='fan_in',
                    nonlinearity='relu')
        sd = {}
        for k, v in shell.state_dict().items():
            v = v.detach().clone().to(device)
            if mode == "bf16" and v.dim() == 4:
                v = v.contiguous(memory_format=torch.channels_last)
            sd[k] = v
        params = []
        for k, v in sd.items():
            if v.is_floating_point() and "running" not in k:
                v.requires_grad_(True)
                params.append(v)
        opt = torch.optim.SGD(params, lr=1e-2, momentum=0.9, weight_decay=5e-4)
        imgs, gts = synth_batch(n, h, w, 7)
        imgs, gts = imgs.to(device), gts.to(device)
        if mode == "bf16":
            imgs = imgs.contiguous(memory_format=torch.channels_last)
        min_kept = n * h * w // 16
        stats = {}

        def one():
            opt.zero_grad()
            if mode == "bf16":
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    lo, _ = torch_ref.bisenet_r18_forward(imgs, sd, 1e-5, 0.1, True, stats)
                lo = [l.float() for l in lo]
                import torch.nn.functional as F
                loss = 0
                for l, sc in zip(lo, (16, 8, 8)):   # losses in fp32, as autocast would run softmax / CE
                    loss = loss + torch_ref.ohem_ce(F.interpolate(l, scale_factor=sc, mode="bilinear", align_corners=True),
                                                    gts, IGNORE, 0.7, min_kept)
            else:
                loss, _ = torch_ref.bisenet_r18_loss(imgs, gts, sd, min_kept, stats=stats)
            loss.backward()
            opt.step()
            return loss

        for _ in range(warmup):
            one()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = one()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        return dict(value=n / (ms / 1000.0), unit="images/sec", ms_per_step=ms, batch=n, steps=steps, warmup=warmup,
                    final_loss=float(loss))
    finally:
        torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        torch.cuda.empty_cache()


def run_eval_bench(args, device):
    """SURVEY §8 f2: evaluator forward throughput — BiSeNet-R18 in eval mode (main head, x8 bilinear, log_softmax;
    network.py:110-111) on whole Cityscapes frames (1024 x 2048), the libtsb path with the BatchNorm folded into the conv
    operands vs the same path un-folded vs the oracle restatement of the reference eval forward on cuDNN (fp32 and bf16
    autocast + channels_last). Not part of the driver's contract: a secondary line (profiles/)."""
    import torch.nn.functional as F
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.seg_opr import seg_oprs
    from torchseg_b200.utils.init_func import init_weight
    from oracle import torch_ref
    n, h, w = args.batch, 1024, 2048
    torch.manual_seed(12345)
    model = BiSeNet(NUM_CLASSES, False, None, None, torch.nn.BatchNorm2d)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, torch.nn.BatchNorm2d, 1e-5, 0.1, mode='fan_in',
                nonlinearity='relu')
    sd = {k: v.detach().clone().to(device) for k, v in model.state_dict().items()}
    model.to(device)
    torchseg_b200.prepare_model(model)
    model.eval()
    x = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(3)).to(device)

    def timeit(fn, steps):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        return dict(value=n / (ms / 1000.0), unit="images/sec", ms_per_batch=ms)

    res = {}
    with torch.no_grad():
        for fold in (True, False):
            seg_oprs.EVAL_FOLD_BN = fold
            res["folded_bn" if fold else "unfolded_bn"] = timeit(lambda: model(x), args.steps)
        seg_oprs.EVAL_FOLD_BN = True

        def ref(mode):
            def f():
                xx = x.contiguous(memory_format=torch.channels_last) if mode == "bf16" else x
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
                    lo, _ = torch_ref.bisenet_r18_forward(xx, sd, training=False)
                return F.log_softmax(F.interpolate(lo[2].float(), scale_factor=8, mode="bilinear", align_corners=True), dim=1)
            return f
        torch.backends.cudnn.benchmark = True
        for mode in ("fp32", "bf16"):
            torch.backends.cudnn.allow_tf32 = mode != "fp32"
            res["reference_cudnn_" + mode] = timeit(ref(mode), max(3, args.steps // 2))
    best_ref = max(res["reference_cudnn_fp32"]["value"], res["reference_cudnn_bf16"]["value"])
    line = {"metric": "images/sec evaluator forward (1024x2048, 19-class, eval-mode BiSeNet-R18)", "value": res["folded_bn"]["value"],
            "unit": "images/sec", "n_gpus": 1, "steps": args.steps, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": "BiSeNet-R18 eval forward incl. x8 upsample + log_softmax, whole 1024x2048 frames", "batch": n},
            "detail": res, "speedup_folding": res["folded_bn"]["value"] / res["unfolded_bn"]["value"],
            "speedup_vs_best_reference_gpu": res["folded_bn"]["value"] / best_ref}
    print(json.dumps(line))


def run_pipeline_bench(args, device):
    """SURVEY §8 f4: the device input pipeline (tsb_train_preprocess / tsb_edge_labels behind TrainPreGPU) on a batch of
    decoded Cityscapes-size frames, against the cv2 sequence the reference's TrainPre runs per sample on one host core
    (dataloader.py:16-33; the reference uses 24 worker processes). Secondary line (profiles/)."""
    import random
    import numpy as np
    from torchseg_b200.utils.gpu_pipeline import TrainPreGPU
    n = BATCH_PER_GPU
    mean, std = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
    rng = np.random.default_rng(0)
    frames = [rng.integers(0, 256, (1024, 2048, 3), dtype=np.uint8) for _ in range(n)]
    gts = [rng.integers(0, 19, (1024, 2048), dtype=np.uint8) for _ in range(n)]
    for g in gts:
        for _ in range(40):
            y0, x0 = rng.integers(0, 1000), rng.integers(0, 2000)
            g[y0:y0 + rng.integers(20, 300), x0:x0 + rng.integers(20, 500)] = rng.integers(0, 19)
    fd = [torch.from_numpy(f).to(device) for f in frames]
    gd = [torch.from_numpy(g).to(device) for g in gts]
    out = {}
    peaks = load_peaks()
    for name, crop, scales, edge in (("bisenet_1024", (1024, 1024), [0.75, 1, 1.25, 1.5, 1.75, 2.0], False),
                                     ("dfn_800_edge_labels", (800, 800), [0.5, 0.75, 1, 1.5, 1.75, 2.0], True)):
        pre = TrainPreGPU(mean, std, crop, scales, device, bgr_input=True, edge_labels=edge)
        random.seed(1)
        params = [pre.draw((1024, 2048)) for _ in range(n)]
        for _ in range(3):
            res = pre(fd, gd, params)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            res = pre(fd, gd, params)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        out_bytes = sum(t.numel() * t.element_size() for t in res)
        # algorithmic bytes: every output element written once + the source pixels of the crop window read once
        src_bytes = sum(min(p["sh"], crop[0]) * min(p["sw"], crop[1]) / ((p["sh"] / 1024.0) * (p["sw"] / 2048.0)) * 4 for p in params)
        entry = dict(value=n / (ms / 1000.0), unit="images/sec", ms_per_batch=ms, batch=n,
                     algorithmic_gb_per_s=(out_bytes + src_bytes) / ms / 1e6, hbm_peak_gb_per_s=peaks["hbm_gbs"])
        # the cv2 sequence of the reference TrainPre on one host core, same parameters (2 samples)
        try:
            import cv2
            cv2.setNumThreads(1)
            k7 = cv2.getStructuringElement(cv2.MORPH_RECT, (7, 7))
            t0 = time.perf_counter()
            for i in range(2):
                p, img, gt = params[i], frames[i][:, :, ::-1], gts[i]
                if p["flip"]:
                    img, gt = cv2.flip(img, 1), cv2.flip(gt, 1)
                img = cv2.resize(img, (p["sw"], p["sh"]), interpolation=cv2.INTER_LINEAR)
                gt = cv2.resize(gt, (p["sw"], p["sh"]), interpolation=cv2.INTER_NEAREST)
                if edge:
                    g0 = gt.copy()
                    g0[gt == 255] = 0
                    cgt = cv2.dilate(cv2.Canny(g0, 5, 5, apertureSize=7), k7)
                x = ((img.astype(np.float32) / 255.0) - mean) / std
                x = x[p["pos_h"]:p["pos_h"] + crop[0], p["pos_w"]:p["pos_w"] + crop[1]]
                x = np.ascontiguousarray(x.transpose(2, 0, 1)).astype(np.float32)
            entry["cv2_one_core_images_per_sec"] = 2 / (time.perf_counter() - t0)
        except ImportError:
            pass
        out[name] = entry
    line = {"metric": "images/sec training input pipeline (1024x2048 uint8 frames -> fp32 NCHW crop + int64 labels)",
            "value": out["bisenet_1024"]["value"], "unit": "images/sec", "n_gpus": 1, "steps": args.steps, "dtype": "u8",
            "data": "synthetic", "config": {"workload": "TrainPre on the device: mirror, cv2-exact scale, normalize, crop/pad (+ DFN border labels)",
                                            "batch": n}, "detail": out}
    print(json.dumps(line))


def pick_threads():
    """torch CPU ops do not scale to every hardware thread of a big host: calibrate on a tiny step and use the
    fastest of {all, 64, 32, 16} threads (reported as `cores`)."""
    n_all = os.cpu_count() or 1
    cands = sorted({c for c in (n_all, 64, 32, 16) if c <= n_all}, reverse=True)
    if len(cands) == 1:
        return cands[0]
    best, best_ips = cands[0], -1.0
    for c in cands:
        ips, _ = cpu_reference_steps(2, 128, 128, 1, 1, c)
        if ips > best_ips:
            best, best_ips = c, ips
    return best


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = pick_threads()
    n, hw = CPU_SAMPLE_BATCH, 1024
    # every one of the K timed steps (and W warm-up steps) is ONE step of the bounded sample: batch 2 @ 1024x1024, the
    # reference's own per-GPU batch (config.py:82 / dataloader.py:53), ~3 s of CPU work each
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    ips, _ = cpu_reference_steps(n, hw, hw, steps, warmup, threads)
    sample = "oracle port of the reference step (fp32 NCHW torch.nn lowering), batch %d @ %dx%d per step, %d warm-up + %d timed steps, %d threads" % (
        n, hw, hw, warmup, steps, threads)
    line = dict(impl="reference", metric=METRIC, value=ips, unit="images/sec", n_gpus=args.gpus, steps=steps,
                warmup=warmup, ms_per_step=1000.0 * n / ips, higher_is_better=True, scaling="weak", vs_baseline=None,
                dtype="f32", data="synthetic",
                config=dict(workload=WORKLOAD, batch_per_step=n, device="host CPU (bounded sample of the same workload)"),
                cpu_baseline=dict(value=ips, unit="images/sec", cores=threads, kind="port", sample=sample),
                e2e=dict(value=ips, unit="images/sec", h2d_bytes_per_step=0, d2h_bytes_per_step=0))
    print(json.dumps(line))


# ------------------------------------------------------------------------------------------------ outputs
DUMP_PARAM_SAMPLE = 1 << 20   # parameter entries written by --dump-outputs (fixed seed → same entries every run)


def dump_outputs(out_dir, loss, model):
    """What the timed step hands back: its loss, and the parameters it updated (a fixed, seeded sample, fp32)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    params = torch.cat([p.detach().float().reshape(-1) for p in model.parameters()]).cpu().numpy()
    idx = np.sort(np.random.default_rng(0).choice(params.size, min(DUMP_PARAM_SAMPLE, params.size), replace=False))
    np.save(os.path.join(out_dir, "loss.npy"), np.array([loss], dtype=np.float32))
    np.save(os.path.join(out_dir, "params_sample.npy"), params[idx].astype(np.float32))
    np.save(os.path.join(out_dir, "params_sample_index.npy"), idx.astype(np.float64))


# ------------------------------------------------------------------------------------------------ main arm
def main():
    global BATCH_PER_GPU, MODEL, H, W, NUM_CLASSES, IGNORE, STEP_GFLOP_PER_IMG, METRIC, WORKLOAD
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--batch", type=int, default=BATCH_PER_GPU, help="per-GPU batch (BASELINE: 16)")
    ap.add_argument("--model", default="bisenet", choices=["bisenet", "pspnet", "psanet", "dfn"],
                    help="bisenet = BASELINE configs[1] (the metric); pspnet / dfn = secondary lines (SURVEY C3 / C4)")
    ap.add_argument("--size", type=int, default=0, help="input size override (pspnet default 480, the reference shape)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-graph", dest="graph", action="store_false",
                    help="single GPU: time eager launches only (default: the step is ONE CUDA graph replay, "
                         "engine.graph.GraphedTrainStep; the eager time is reported beside it)")
    ap.add_argument("--pipeline", action="store_true", help="secondary line: device input pipeline throughput, 1 GPU")
    ap.add_argument("--eval", action="store_true", help="secondary line: evaluator forward throughput (BN folding), 1 GPU")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (loss, a fixed seeded sample of "
                         "the updated parameters) to DIR/<name>.npy")
    ap.add_argument("--default-stream", action="store_true",
                    help="run on the legacy default stream (default: a non-blocking side stream, which whole-step graph capture needs)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference_arm(args)

    import torch.distributed as dist
    from torchseg_b200 import _lib, ops
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if not torch.cuda.is_available():
        raise RuntimeError("bench.py (impl b200) needs a CUDA device: the hot path has no CPU fallback")
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", init_method="env://", device_id=device)
    if args.pipeline:
        return run_pipeline_bench(args, device)
    if args.eval:
        if args.batch == BATCH_PER_GPU:
            args.batch = 4
        return run_eval_bench(args, device)
    if not args.default_stream:
        # everything (warm-up, timed regions, autograd's accumulation streams) lives on ONE non-default stream: a stream
        # capture is invalidated by any work that touches the legacy default stream
        torch.cuda.set_stream(torch.cuda.Stream(device=device))
    warmup = max(3, args.warmup)
    BATCH_PER_GPU = args.batch
    if args.model == "pspnet":
        MODEL, NUM_CLASSES, IGNORE = "pspnet", 150, -1
        H = W = args.size or 480
        # BASELINE.md §2: 529.62 GF fwd @480^2 (step 1588.7); 1190.8 GF fwd @713^2 (90x90 feature map) ⇒ step 3 x 1190.8 - 0.45
        STEP_GFLOP_PER_IMG = (3 * 1190.8 - 0.45) if H == 713 else 1588.7 * (H * W) / (480.0 * 480.0)
        METRIC = "images/sec training step (%dx%d, 150-class)" % (H, W)
        WORKLOAD = "PSPNet-R101_v1c dilated-8 train step, %dx%d, 150-class CE (BASELINE configs[2] family, reference shape 480)" % (H, W)
    elif args.model == "psanet":
        MODEL, NUM_CLASSES, IGNORE = "psanet", 150, -1
        H = W = args.size or 480    # the PSA head needs exactly 60x60 = 3600 positions (psanet network.py:88): 473..480
        # SURVEY §8d: conv 590.03 GF (@480; 589.58 @473) + bmm 26.5 GF fwd
        STEP_GFLOP_PER_IMG = 3 * ((589.58 if H == 473 else 590.03) + 26.5) - 2 * 0.10
        METRIC = "images/sec training step (%dx%d, 150-class)" % (H, W)
        WORKLOAD = "PSANet-R101_v1c dilated-8 train step, %dx%d, 150-class CE (SURVEY C5 / BASELINE configs[4] at 473); conv + PSA bmm FLOPs" % (H, W)
    elif args.model == "dfn":
        MODEL = "dfn"
        H = W = args.size or 1024
        # SURVEY §8d: 2217.6 GF fwd conv @1024^2; step = 3x - 2x the image-input conv (3->32 3x3/2: 0.453 GF)
        STEP_GFLOP_PER_IMG = (3 * 2217.6 - 2 * 0.453) * (H * W) / (1024.0 * 1024.0)
        METRIC = "images/sec training step (%dx%d, 19-class + border)" % (H, W)
        WORKLOAD = "DFN-R101_v1c train step, %dx%d, 4x CE + 0.1 * 4x focal (SURVEY C4; reference shape 800, 4 img/GPU)" % (H, W)
    elif args.size:
        H = W = args.size

    model, ddp, opt, lr_policy = build_b200(device, world)
    host_batch = synth_batch(BATCH_PER_GPU, H, W, 100 + rank, pin=True)
    dev_batch = tuple(t.to(device) for t in host_batch)
    keys = ("data", "label", "aux_label")[:len(host_batch)]

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        t = torch.tensor([ms], dtype=torch.float64, device=device)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def set_lr(it_):
        lr = lr_policy.get_lr(it_)
        for i, g in enumerate(opt.param_groups):
            g['lr'] = lr if i < 2 else lr * 10  # train.py:136-139

    it = 0
    for _ in range(warmup):
        train_step(model, ddp, opt, lr_policy, it, *dev_batch)   # (no reference to the loss is kept: a live autograd graph
        it += 1                                                    # of an eager step invalidates a later whole-step capture)

    def timed_eager(nsteps):
        nonlocal it
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = _lib.launch_count()
        with ClockSampler(local) as clk_:
            e0.record()
            for _ in range(nsteps):
                loss_ = train_step(model, ddp, opt, lr_policy, it, *dev_batch)
                it += 1
            e1.record()
            barrier()
        return max_over_ranks(e0.elapsed_time(e1)), clk_, _lib.launch_count() - n0, loss_

    # ---------------- timed region 1 (`value`), CLEAN: no event instrumentation, inputs resident in HBM.
    # The whole step (zero_grad → forward → backward → [bucketed NCCL gradient all-reduce on the side stream, NVLink SyncBN
    # exchanges] → fused SGD) is ONE CUDA graph replay (torchseg_b200.engine.graph.GraphedTrainStep) unless --no-graph /
    # capture is unavailable; the eager-launch time of the same step is measured and reported beside it.
    # eager launches first (DDP in its overlapped mode), then the graph: no autograd graph of an eager step may be alive
    # when the capture starts, so only the loss VALUE is kept
    ms_eager, clk_eager, launches_eager, loss = timed_eager(args.steps)
    ms, clk, launches, final_loss = ms_eager, clk_eager, launches_eager, float(loss.item())
    del loss
    gstep = None
    if args.graph and (world == 1 or os.environ.get("TSB_BENCH_GRAPH_MULTI", "1") != "0"):
        from torchseg_b200.engine.graph import GraphedTrainStep
        set_lr(it)
        gstep = GraphedTrainStep(model, opt, dev_batch, warmup=2, ddp=ddp)
        ok = torch.tensor([1.0 if gstep.graph is not None else 0.0], device=device)
        if world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)     # all ranks replay, or none does
        if float(ok.item()) < 1.0:
            sys.stderr.write("bench: CUDA graph capture unavailable (%s); eager step timed instead\n" % gstep.error)
            gstep = None
    if gstep is not None:
        static_in = gstep.static_inputs
        for _ in range(2):
            set_lr(it)
            loss = gstep(*static_in)
            it += 1
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with ClockSampler(local) as clk_g:
            e0.record()
            for _ in range(args.steps):
                set_lr(it)
                loss = gstep(*static_in)      # inputs already in the graph's static buffers: no copy
                it += 1
            e1.record()
            barrier()
        ms, clk = max_over_ranks(e0.elapsed_time(e1)), clk_g
        launches = gstep.launches_per_step * args.steps
        final_loss = float(loss.item())
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, final_loss, model)

    # ---------------- measurement pass B (separate, NOT part of `value`): every conv launch bracketed by CUDA events on
    # the launch stream → roofline.achieved = algorithmic conv FLOPs / summed conv kernel time
    prof_steps = min(args.steps, 5)
    ops.conv_prof.enable()
    timed_eager(prof_steps)
    prof = ops.conv_prof.collect()
    ops.conv_prof.disable()

    def run_step(it_, *inputs):
        if gstep is not None:
            set_lr(it_)
            return gstep(*inputs)
        return train_step(model, ddp, opt, lr_policy, it_, *inputs)

    # ---------------- timed region 2: end to end through the public API with HOST buffers: every step's inputs are
    # copied from pinned host memory (CudaPrefetcher: side-stream copy of batch i+1 under step i) and every step's
    # loss is read back to the host (async D2H into pinned memory, value consumed one step later)
    from torchseg_b200.utils.prefetch import CudaPrefetcher

    def host_batches(n):
        for _ in range(n):
            yield dict(zip(keys, host_batch))

    loss_host = torch.zeros(args.steps, dtype=torch.float32).pin_memory()
    # one untimed e2e step warms the pipeline (device slots allocated, first batch in flight); inside the timed region
    # exactly one H2D batch copy is issued per step (the copy of step i+1 overlaps the compute of step i)
    loader = CudaPrefetcher(host_batches(args.steps + 2), device)
    mb = loader.next()
    run_step(it, *[mb[k] for k in keys])
    it += 1
    barrier()
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e2.record()
    for k in range(args.steps):
        mb = loader.next()                                       # train.py:119-124
        loss = run_step(it, *[mb[k_] for k_ in keys])
        it += 1
        loss_host[k:k + 1].copy_(loss.detach().reshape(1), non_blocking=True)   # train.py:146 (per-iteration loss read)
    e3.record()
    barrier()
    ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    assert bool(torch.isfinite(loss_host).all()), "non-finite loss in the e2e region"

    step_launch = "one CUDA graph replay per step (GraphedTrainStep)" if gstep is not None else "eager launches"
    if gstep is not None:
        gstep.release()    # a live graph that captured NCCL kernels blocks the communicator teardown
    if world > 1:      # all collective work is done: ranks > 0 leave, rank 0 reports (no rank spins in a barrier)
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        peaks = load_peaks()
        n_img = BATCH_PER_GPU * world * args.steps
        value = n_img / (ms / 1000.0)
        e2e_v = n_img / (ms_e2e / 1000.0)
        # ALGORITHMIC conv FLOPs of the step (SURVEY §8d figure x images of this rank) over the measured duration of all
        # conv launches of the instrumented pass. prof["flops"] counts the launched shapes, which include the zero-padded
        # channels of DFN's ragged layers (and is identical to the algorithmic figure for BiSeNet / PSPNet).
        algo_flops = STEP_GFLOP_PER_IMG * 1e9 * BATCH_PER_GPU * prof_steps
        conv_tf = min(prof["flops"], algo_flops) / max(prof["ms"], 1e-9) / 1e9
        traffic = None
        traffic_src = None
        for cand in ("r02_conv_traffic.json", "r01_conv_traffic.json"):
            tpath = os.path.join(ROOT, "profiles", cand)
            if os.path.exists(tpath) and MODEL == "bisenet":  # DRAM bytes of the same launches from the committed ncu pass (per step)
                traffic = json.load(open(tpath)).get("conv_dram_bytes_per_step")
                traffic_src = "profiles/" + cand
                break
        line = {
            "metric": METRIC, "value": value, "unit": "images/sec", "n_gpus": world, "steps": args.steps,
            "warmup": warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": WORKLOAD,
                       "batch_per_gpu": BATCH_PER_GPU, "global_batch": BATCH_PER_GPU * world, "parallelism": "dp%d" % world,
                       "sync_bn": world > 1, "optimizer": "fused flat SGD (momentum 0.9, poly LR, reference wd / lr groups)",
                       "l2_policy": "inputs larger than L2 (activations >> 50 MB per step), no explicit flush",
                       "final_loss": final_loss,
                       "step_launch": step_launch,
                       "sync_bn_exchange": (None if world == 1 else ("NVLink peer-memory kernel (tsb_p2p_allreduce_sum)" if ops._sync.get("p2p") is not None else "NCCL all-reduce per layer")),
                       "eager_ms_per_step": ms_eager / args.steps,
                       "step_conv_gflop_per_img": STEP_GFLOP_PER_IMG,
                       "frac_of_conv_flop_roofline": value / world * STEP_GFLOP_PER_IMG / 1e3 / peaks["tflops"]},
            "e2e": {"value": e2e_v, "unit": "images/sec",
                    "h2d_bytes_per_step": int(sum(t.numel() * t.element_size() for t in host_batch)), "d2h_bytes_per_step": 4,
                    "input_pipeline": "pinned host buffers, side-stream prefetch (torchseg_b200.utils.prefetch.CudaPrefetcher)"},
            "gpu_launches": int(launches),
            "clocks": clk.summary(),
            "roofline": {"bound": "tensor", "achieved": conv_tf, "peak": peaks["tflops"], "unit": "TFLOP/s",
                         "frac": conv_tf / peaks["tflops"], "traffic": traffic,
                         "traffic_note": "dram__bytes_read+write summed over the conv launches of ONE step (%s); algorithmic minimum ~5.9 GB/step" % traffic_src,
                         "flops_per_step": min(prof["flops"], algo_flops) / prof_steps,
                         "launched_flops_per_step": prof["flops"] / prof_steps,
                         "kernel": "wgmma implicit-GEMM conv kernels (igemm_v2_kernel fprop/dgrad/stem + wgrad kernels), all launches of the step",
                         "launches": prof["launches"], "kernel_ms_per_step": prof["ms"] / prof_steps,
                         "measured_in": "separate instrumented pass of %d eager steps (not the `value` region)" % prof_steps,
                         "peak_source": peaks["src"]},
        }
        if world == 1 and not args.no_cpu_baseline and MODEL == "bisenet":
            # the reference step on THIS GPU under stock PyTorch + cuDNN (SURVEY §8d last row): the numbers the kernels
            # must beat; strict fp32 is the parity configuration, bf16 autocast + channels_last the fastest stock one
            ref_gpu = {}
            nb = BATCH_PER_GPU
            for mode in ("fp32", "bf16"):
                try:
                    ref_gpu[mode] = gpu_reference_steps(device, nb, H, W, 3, 2, mode)
                except torch.OutOfMemoryError:
                    torch.cuda.empty_cache()
                    nb = max(2, nb // 2)
                    ref_gpu[mode] = gpu_reference_steps(device, nb, H, W, 3, 2, mode)
            best = max(v["value"] for v in ref_gpu.values())
            line["reference_gpu"] = {"kind": "port", "what": "oracle restatement of the reference step (stock torch.nn + cuDNN, cudnn.benchmark=True, torch.optim.SGD) on the same GPU",
                                     "fp32": ref_gpu["fp32"], "bf16_autocast_channels_last": ref_gpu["bf16"],
                                     "speedup_vs_fp32": value / ref_gpu["fp32"]["value"], "speedup_vs_best": value / best}
            threads = pick_threads()
            ips, _ = cpu_reference_steps(CPU_SAMPLE_BATCH, 1024, 1024, 2, 1, threads)
            line["cpu_baseline"] = {"value": ips, "unit": "images/sec", "cores": threads, "kind": "port",
                                    "sample": "oracle port of the reference step, batch %d @ 1024x1024, 1 warm-up + 2 timed steps" % CPU_SAMPLE_BATCH}
        print(json.dumps(line))


if __name__ == "__main__":
    main()
