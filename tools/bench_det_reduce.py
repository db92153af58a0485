"""Per-call time of the ordered slot sums (tsb_det_reduce) of one BiSeNet-R18 training step (bench.py's model at
16 x 1024^2), old kernel against new, CUDA events.

    python tools/bench_det_reduce.py [--batch 16] [--reps 200] [--rounds 5] [--out DIR]

1. One training step is captured into a CUDA graph and its kernel nodes are read back through the driver API: every
   det_reduce launch gives its (nparts, n, stride) and which kernel ran it.
2. For every distinct shape, R launches of the grid-wide `det_reduce_kernel` as the previous commit ran it for every
   n (one thread per output, tsb_grid_for(n, 256, 8) CTAs of 256), and R launches of tsb_det_reduce as it dispatches
   now, are each captured into a CUDA graph; the two graphs are replayed alternately, `--rounds` times each, and the
   best round is kept. For n == stride with an even n of at most 2048 (a statistics pair that tsb_det_reduce_pair now
   sums in one launch) the two launches over n / 2 outputs that the previous commit made are timed as well.
3. Reported per shape: µs per call, GB/s of slot bytes (nparts · n · 4 B read) and the 4-cycle-per-add chain floor
   nparts · 4 / f_max (f_max = the card's maximum SM clock), and the per-step totals.
Writes DIR/det_reduce.json with the card name and power limit read in the same run."""
import argparse
import collections
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from bench_stem import gpu_info  # noqa: E402


class KernelNodeParams(ctypes.Structure):
    """CUDA_KERNEL_NODE_PARAMS_v2 (cuda.h)"""
    _fields_ = [("func", ctypes.c_void_p), ("gridDimX", ctypes.c_uint), ("gridDimY", ctypes.c_uint),
                ("gridDimZ", ctypes.c_uint), ("blockDimX", ctypes.c_uint), ("blockDimY", ctypes.c_uint),
                ("blockDimZ", ctypes.c_uint), ("sharedMemBytes", ctypes.c_uint),
                ("kernelParams", ctypes.POINTER(ctypes.c_void_p)), ("extra", ctypes.c_void_p),
                ("kern", ctypes.c_void_p), ("ctx", ctypes.c_void_p)]


def _cu():
    cu = ctypes.CDLL("libcuda.so.1")
    cu.cuGraphGetNodes.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]
    cu.cuGraphNodeGetType.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
    cu.cuGraphKernelNodeGetParams_v2.argtypes = [ctypes.c_void_p, ctypes.POINTER(KernelNodeParams)]
    cu.cuFuncGetName.argtypes = [ctypes.POINTER(ctypes.c_char_p), ctypes.c_void_p]
    cu.cuLaunchKernel.argtypes = [ctypes.c_void_p] + [ctypes.c_uint] * 6 + [ctypes.c_uint, ctypes.c_void_p,
                                                                              ctypes.c_void_p, ctypes.c_void_p]
    return cu


def _check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed: CUresult %d" % (what, rc))


def step_calls(cu, batch):
    """[(kernel name, nparts, n, stride)] of every det_reduce launch of one captured BiSeNet-R18 step (graph node order),
    and the CUfunction of the grid-wide kernel"""
    dev = torch.device("cuda:0")
    bench.BATCH_PER_GPU = batch
    model, ddp, opt, lrp = bench.build_b200(dev, 1)
    imgs, gts = bench.synth_batch(batch, bench.H, bench.W, 100)
    imgs, gts = imgs.to(dev), gts.to(dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for it in range(2):
            bench.train_step(model, ddp, opt, lrp, it, imgs, gts)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    opt.push_hyperparams()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        bench.train_step(model, ddp, opt, lrp, 2, imgs, gts)
    graph = g.raw_cuda_graph()
    num = ctypes.c_size_t(0)
    _check(cu.cuGraphGetNodes(graph, None, ctypes.byref(num)), "cuGraphGetNodes")
    nodes = (ctypes.c_void_p * num.value)()
    _check(cu.cuGraphGetNodes(graph, nodes, ctypes.byref(num)), "cuGraphGetNodes")
    calls, grid_fn = [], None
    for node in nodes:
        t = ctypes.c_int(-1)
        _check(cu.cuGraphNodeGetType(node, ctypes.byref(t)), "cuGraphNodeGetType")
        if t.value != 0:   # CU_GRAPH_NODE_TYPE_KERNEL
            continue
        p = KernelNodeParams()
        _check(cu.cuGraphKernelNodeGetParams_v2(node, ctypes.byref(p)), "cuGraphKernelNodeGetParams")
        name = ctypes.c_char_p()
        _check(cu.cuFuncGetName(ctypes.byref(name), p.func), "cuFuncGetName")
        name = name.value.decode()
        if "det_reduce" not in name:
            continue
        a = p.kernelParams   # (out, parts, nparts, n, stride)
        nparts = ctypes.cast(a[2], ctypes.POINTER(ctypes.c_int))[0]
        n = ctypes.cast(a[3], ctypes.POINTER(ctypes.c_longlong))[0]
        stride = ctypes.cast(a[4], ctypes.POINTER(ctypes.c_longlong))[0]
        kind = "cols" if "cols" in name else "grid"
        if kind == "grid":
            grid_fn = p.func
        calls.append((kind, nparts, n, stride))
    g.reset()
    del model, ddp, opt, g
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return calls, grid_fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=200, help="launches per captured graph")
    ap.add_argument("--rounds", type=int, default=5, help="alternated replays of each graph; the best is kept")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_det_reduce.py times kernels on the GPU"
    torch.cuda.set_device(0)
    from torchseg_b200 import _lib
    lib = _lib.lib()
    lib.tsb_det_reduce.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_longlong,
                                   ctypes.c_void_p]
    cu = _cu()
    info = gpu_info()
    try:
        fmax_ghz = float(info["max_sm_clock"].split()[0]) / 1e3
    except Exception:  # noqa: BLE001
        fmax_ghz = 1.98
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    calls, grid_fn = step_calls(cu, args.batch)
    if grid_fn is None:
        raise RuntimeError("the step launched no grid-wide det_reduce_kernel: nothing to time the old form with")
    shapes = collections.Counter((c[1], c[2], c[3]) for c in calls)
    kinds = {(c[1], c[2], c[3]): c[0] for c in calls}

    def old_launch(out, parts, nparts, n, stride):
        grid = min(max((n + 255) // 256, 1), sms * 8)
        vals = [ctypes.c_void_p(out), ctypes.c_void_p(parts), ctypes.c_int(nparts), ctypes.c_longlong(n),
                ctypes.c_longlong(stride)]
        arr = (ctypes.c_void_p * 5)(*[ctypes.cast(ctypes.byref(v), ctypes.c_void_p) for v in vals])
        _check(cu.cuLaunchKernel(grid_fn, grid, 1, 1, 256, 1, 1, 0, torch.cuda.current_stream().cuda_stream, arr, None),
               "cuLaunchKernel")

    def new_launch(out, parts, nparts, n, stride):
        rc = lib.tsb_det_reduce(out, parts, nparts, n, stride, torch.cuda.current_stream().cuda_stream)
        if rc != 0:
            raise RuntimeError(lib.tsb_last_error().decode())

    def graph_of(fn):   # the launches go to the capture stream, the current stream inside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(args.reps):
                fn()
        return g

    def time_graph(g):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.reps   # µs per call

    rows = []
    gen = torch.Generator(device="cuda").manual_seed(0)
    for (nparts, n, stride), count in sorted(shapes.items(), key=lambda kv: (-kv[0][0] * kv[0][1], kv[0])):
        parts = torch.randn(nparts * stride, device="cuda", generator=gen)
        out = torch.zeros(n, device="cuda")
        po, pp = out.data_ptr(), parts.data_ptr()
        forms = {"old": graph_of(lambda: old_launch(po, pp, nparts, n, stride)),
                 "new": graph_of(lambda: new_launch(po, pp, nparts, n, stride))}
        pair = n == stride and n % 2 == 0 and n <= 2048
        if pair:
            h = n // 2

            def old_pair():
                old_launch(po, pp, nparts, h, stride)
                old_launch(po + 4 * h, pp + 4 * h, nparts, h, stride)
            forms["old_two_halves"] = graph_of(old_pair)
        best = {k: float("inf") for k in forms}
        for _ in range(args.rounds):
            for k, g in forms.items():
                time_graph(g)                        # the first replay of a round warms the shape
                best[k] = min(best[k], time_graph(g))
        floor_us = nparts * 4 / (fmax_ghz * 1e3)
        row = dict(nparts=nparts, n=n, stride=stride, calls=count, kernel_now=kinds[(nparts, n, stride)],
                   old_us=round(best["old"], 3), new_us=round(best["new"], 3),
                   old_gbs=round(nparts * n * 4 / best["old"] / 1e3, 1), new_gbs=round(nparts * n * 4 / best["new"] / 1e3, 1),
                   chain_floor_us=round(floor_us, 3))
        if pair:
            row["old_two_halves_us"] = round(best["old_two_halves"], 3)
        rows.append(row)
        print("nparts %5d n %8d stride %8d x%3d [%s]: old %8.2f us%s, new %8.2f us (%7.1f GB/s), chain floor %.2f us" % (
            nparts, n, stride, count, row["kernel_now"], row["old_us"],
            " (two halves %.2f us)" % row["old_two_halves_us"] if pair else "", row["new_us"], row["new_gbs"], floor_us))
        del forms
    tot_new = sum(r["new_us"] * r["calls"] for r in rows)
    tot_old = sum(r.get("old_two_halves_us", r["old_us"]) * r["calls"] for r in rows)
    print("%s: %d det_reduce launches per step; new %.1f us; old %.1f us (pairs as two launches)" % (
        info.get("name"), len(calls), tot_new, tot_old))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "det_reduce.json"), "w") as f:
            json.dump(dict(gpu=info, batch=args.batch, reps=args.reps, rounds=args.rounds, launches=len(calls),
                           step_new_us=tot_new, step_old_us=tot_old, shapes=rows), f, indent=1)


if __name__ == "__main__":
    main()
