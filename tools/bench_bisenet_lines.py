"""Benchmark of the BiSeNet lines R18.speed, X39.speed and R101 on one GPU: training img/s and batch-1 inference FPS.

    python tools/bench_bisenet_lines.py [--lines r18_speed,x39_speed,r101] [--steps 20] [--warmup 5]
                                        [--ref-steps 10] [--ref-warmup 3] [--no-ref] [--infer-iters 100]
                                        [--dump-outputs DIR]

Prints one JSON line with, per line:
  * training at the reference shape (R101 16x3x1024², each .speed line 16x3x768x1536 with 96x192 labels and the .speed
    min_kept = batch·H·W // (16·8²)): the graph-replayed libtsb step (engine.graph.GraphedTrainStep), img/s and
    ms/step from CUDA events, and the step's peak memory (torch.cuda.max_memory_allocated);
  * the same step for the oracle (tests/bisenet_lines_oracle.py: the reference's stock torch.nn lowering) on cuDNN,
    strict fp32 and bf16 autocast + channels_last, as tools/bench_x39.py's reference arms do;
  * for the .speed lines, eval-mode inference (folded BN) at batch 1, 1x3x768x1536 and 1x3x512x1024 (the default of
    the reference's `eval.py -speed`): frames/s eager and as one CUDA-graph replay per frame, and the oracle's eager
    frames/s on cuDNN (fp32 and bf16 autocast);
and the card name, power limit and max SM clock (nvidia-smi, read-only query) of the run.
--dump-outputs DIR writes each line's last timed training loss and a seeded sample of the updated parameters to
DIR/<line>/ (.npy), so two runs can be compared bit for bit.
"""
import argparse
import importlib
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_x39 import IGNORE, NUM_CLASSES, dump_outputs, gpu_info, synth_batch, time_events  # noqa: E402

BN = torch.nn.BatchNorm2d
# line → (module under torchseg_b200.networks, training shape N, H, W, label down-sampling, takes ohem_criterion)
LINES = {
    "r18_speed": ("bisenet_speed", (16, 768, 1536), 8, True),
    "x39_speed": ("bisenet_x39_speed", (16, 768, 1536), 8, True),
    "r101": ("bisenet_r101", (16, 1024, 1024), 1, False),
}
INFER_SHAPES = [(768, 1536), (512, 1024)]


def _net(line, training, crit=None):
    mod, _, _, two_crit = LINES[line]
    cls = importlib.import_module("torchseg_b200.networks." + mod).BiSeNet
    if two_crit:
        return cls(NUM_CLASSES, training, torch.nn.CrossEntropyLoss(ignore_index=IGNORE) if training else None, crit,
                   None, BN)
    return cls(NUM_CLASSES, training, crit, None, BN)


def _batch(line):
    (n, h, w), d = LINES[line][1], LINES[line][2]
    x, _ = synth_batch(n, h, w, 7)
    _, y = synth_batch(n, h // d, w // d, 8)
    return x, y, n * h * w // (16 * d * d)


def _init(model):
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(12345)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    return model


def _initial_state(line):
    """the training arm's initial weights (same seed, same init), on the host"""
    torch.manual_seed(12345)
    m = _init(_net(line, True))
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def train_arm(dev, line, steps, warmup):
    import torchseg_b200
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import group_weight
    x, y, min_kept = _batch(line)
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(12345)
    ohem = ProbOhemCrossEntropy2d(ignore_label=IGNORE, thresh=0.7, min_kept=min_kept, use_weight=False)
    model = _init(_net(line, True, ohem))
    model.to(dev)
    torchseg_b200.prepare_model(model)
    model.train()
    groups = group_weight([], model.context_path, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    opt = optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)
    x, y = x.to(dev), y.to(dev)
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        step = GraphedTrainStep(model, opt, [x, y], warmup=2)
        if step.graph is None:
            raise RuntimeError("CUDA graph capture failed: %s" % step.error)
        for _ in range(warmup):
            step(x, y)
        torch.cuda.synchronize()
        ms, loss = time_events(lambda: step(x, y), steps)
        loss = float(loss.detach())
        peak = torch.cuda.max_memory_allocated()
        step.release()
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())
    n = x.shape[0]
    return dict(value=n / (ms / 1e3), unit="images/sec", ms_per_step=ms, batch=n, image=list(x.shape[2:]),
                label=list(y.shape[1:]), min_kept=min_kept, steps=steps, warmup=warmup, final_loss=loss,
                launches_per_step=step.launches_per_step, peak_memory_gib=round(peak / 2 ** 30, 2)), model, loss


def _oracle_sd(dev, sd0, mode, grad):
    sd, params = {}, []
    for k, v in sd0.items():
        v = v.detach().clone().to(dev)
        if mode == "bf16" and v.dim() == 4:
            v = v.contiguous(memory_format=torch.channels_last)
        if grad and v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
            params.append(v)
        sd[k] = v
    return sd, params


class _CudnnMode(object):
    """cuDNN benchmark on; 'fp32' strict (TF32 off), 'bf16' with TF32 allowed for what autocast leaves in fp32"""

    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        self.old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.benchmark = True
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = self.mode != "fp32"

    def __exit__(self, *exc):
        torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old
        torch.cuda.empty_cache()


def reference_train_arm(dev, line, steps, warmup, mode, sd0):
    """the oracle step under cuDNN"""
    import bisenet_lines_oracle as tr
    with _CudnnMode(mode):
        sd, params = _oracle_sd(dev, sd0, mode, True)
        opt = torch.optim.SGD(params, lr=1e-2, momentum=0.9, weight_decay=5e-4)
        x, y, min_kept = _batch(line)
        x, y = x.to(dev), y.to(dev)
        if mode == "bf16":
            x = x.contiguous(memory_format=torch.channels_last)
        stats = {}

        def one():
            opt.zero_grad()
            if mode == "bf16":
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    lo, _ = tr.bisenet_forward(line, x, sd, 1e-5, 0.1, True, stats)
                loss = 0
                for l, sc in zip([l.float() for l in lo], tr.LINES[line][1]):
                    loss = loss + tr.ohem_ce(tr.head_up(l, sc), y, IGNORE, 0.7, min_kept)
            else:
                loss, _ = tr.bisenet_loss(line, x, y, sd, min_kept, stats=stats)
            loss.backward()
            opt.step()
            return loss

        for _ in range(warmup):
            one()
        torch.cuda.synchronize()
        ms, loss = time_events(one, steps)
        return dict(value=x.shape[0] / (ms / 1e3), unit="images/sec", ms_per_step=ms, steps=steps, warmup=warmup,
                    final_loss=float(loss.detach()))


def infer_arm(dev, line, iters):
    """eval-mode network (folded BN) at batch 1: frames/s eager and as one CUDA-graph replay per frame"""
    import torchseg_b200
    model = _init(_net(line, False))
    model.to(dev)
    torchseg_b200.prepare_model(model)
    model.eval()
    out = {}
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        for h, w in INFER_SHAPES:
            x = synth_batch(1, h, w, 9)[0].to(dev)
            with torch.no_grad():
                for _ in range(5):
                    model(x)
                torch.cuda.synchronize()
                ms_eager, _ = time_events(lambda: model(x), iters)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    model(x)
            for _ in range(5):
                graph.replay()
            torch.cuda.synchronize()
            ms_graph, _ = time_events(graph.replay, iters)
            del graph
            out["1x3x%dx%d" % (h, w)] = dict(eager_fps=round(1e3 / ms_eager, 1), eager_ms=round(ms_eager, 3),
                                              graph_fps=round(1e3 / ms_graph, 1), graph_ms=round(ms_graph, 3),
                                              iters=iters)
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())
    return out


def reference_infer_arm(dev, line, iters, mode, sd0):
    """the oracle's eval forward (main head, log_softmax) under cuDNN at batch 1, eager"""
    import bisenet_lines_oracle as tr
    out = {}
    with _CudnnMode(mode):
        # the eval network holds no aux heads (heads = [None, None, head])
        sd, _ = _oracle_sd(dev, {k: v for k, v in sd0.items() if not k.startswith(("heads.0.", "heads.1."))}, mode,
                           False)
        for h, w in INFER_SHAPES:
            x = synth_batch(1, h, w, 9)[0].to(dev)
            if mode == "bf16":
                x = x.contiguous(memory_format=torch.channels_last)

            def one():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
                    return tr.bisenet_eval(line, x, sd)

            for _ in range(5):
                one()
            torch.cuda.synchronize()
            ms, _ = time_events(one, iters)
            out["1x3x%dx%d" % (h, w)] = dict(eager_fps=round(1e3 / ms, 1), eager_ms=round(ms, 3), iters=iters)
    return out


def _guard(fn, *args):
    try:
        return fn(*args)
    except torch.cuda.OutOfMemoryError as e:
        torch.cuda.empty_cache()
        return dict(error="out of memory: %s" % str(e).split("\n")[0][:160])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lines", default=",".join(LINES))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=10)
    ap.add_argument("--ref-warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true", help="skip the oracle / cuDNN arms")
    ap.add_argument("--infer-iters", type=int, default=100)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    lines = args.lines.split(",")
    for line in lines:
        if line not in LINES:
            raise SystemExit("unknown line %r (one of %s)" % (line, ", ".join(LINES)))
    if not torch.cuda.is_available():
        raise SystemExit("bench_bisenet_lines measures the GPU and needs a CUDA device")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    result = dict(metric="bisenet_lines", gpu=gpu_info())
    for line in lines:
        row = {}
        row["train_libtsb_graph"], model, loss = train_arm(dev, line, args.steps, args.warmup)
        if args.dump_outputs:
            dump_outputs(os.path.join(args.dump_outputs, line), loss, model)
        del model
        torch.cuda.empty_cache()
        if line != "r101":
            row["infer_libtsb"] = infer_arm(dev, line, args.infer_iters)
            torch.cuda.empty_cache()
        if not args.no_ref:
            sd0 = _initial_state(line)
            for mode in ("fp32", "bf16"):
                row["train_reference_%s" % mode] = _guard(reference_train_arm, dev, line, args.ref_steps,
                                                          args.ref_warmup, mode, sd0)
                if line != "r101":
                    row["infer_reference_%s" % mode] = _guard(reference_infer_arm, dev, line, args.infer_iters, mode,
                                                              sd0)
        result[line] = row
    print(json.dumps(result))


if __name__ == "__main__":
    main()
