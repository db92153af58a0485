"""Micro-benchmark of the conv launches of one BiSeNet-R18 training step (batch 16 @ 1024x1024): every distinct conv
shape with its multiplicity in the step and the passes it runs (F = fprop, with BN statistics where the layer has BN;
D = dgrad; W = wgrad). CUDA events around single launches, L2 flushed before each, median of 10.

Prints µs and TF/s per (shape, pass) and the step-weighted total, comparable with bench.py's
roofline.kernel_ms_per_step. With --out DIR the table is also written to DIR/bench_conv.json.

Usage: python tools/bench_conv.py [--out DIR]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torchseg_b200 import ops

N = 16
# (name, C, H, W, K, R, stride, pad, count in the step, passes, BN statistics in the forward)
STEP = [
    ("spatial 3x3/2 64->64 @512", 64, 512, 512, 64, 3, 2, 1, 1, "FDW", True),
    ("spatial 3x3/2 64->64 @256", 64, 256, 256, 64, 3, 2, 1, 1, "FDW", True),
    ("spatial 1x1 64->128 @128", 64, 128, 128, 128, 1, 1, 0, 1, "FDW", True),
    ("layer1 3x3 64->64 @256", 64, 256, 256, 64, 3, 1, 1, 4, "FDW", True),
    ("layer2.0 3x3/2 64->128 @256", 64, 256, 256, 128, 3, 2, 1, 1, "FDW", True),
    ("layer2.0 ds 1x1/2 64->128 @256", 64, 256, 256, 128, 1, 2, 0, 1, "FDW", True),
    ("layer2/refine 3x3 128->128 @128", 128, 128, 128, 128, 3, 1, 1, 4, "FDW", True),
    ("layer3.0 3x3/2 128->256 @128", 128, 128, 128, 256, 3, 2, 1, 1, "FDW", True),
    ("layer3.0 ds 1x1/2 128->256 @128", 128, 128, 128, 256, 1, 2, 0, 1, "FDW", True),
    ("layer3 3x3 256->256 @64", 256, 64, 64, 256, 3, 1, 1, 3, "FDW", True),
    ("layer4.0 3x3/2 256->512 @64", 256, 64, 64, 512, 3, 2, 1, 1, "FDW", True),
    ("layer4.0 ds 1x1/2 256->512 @64", 256, 64, 64, 512, 1, 2, 0, 1, "FDW", True),
    ("layer4 3x3 512->512 @32", 512, 32, 32, 512, 3, 1, 1, 3, "FDW", True),
    ("global context 1x1 512->128 @1", 512, 1, 1, 128, 1, 1, 0, 1, "FDW", True),
    ("ARM 3x3 512->128 @32", 512, 32, 32, 128, 3, 1, 1, 1, "FDW", True),
    ("ARM 3x3 256->128 @64", 256, 64, 64, 128, 3, 1, 1, 1, "FDW", True),
    ("ARM attention 1x1 128->128 @1", 128, 1, 1, 128, 1, 1, 0, 2, "FDW", True),
    ("refine 3x3 128->128 @64", 128, 64, 64, 128, 3, 1, 1, 1, "FDW", True),
    ("FFM 1x1 256->256 @128", 256, 128, 128, 256, 1, 1, 0, 1, "FDW", True),
    ("FFM attention 1x1 256->64 @1", 256, 1, 1, 64, 1, 1, 0, 1, "FDW", False),
    ("FFM attention 1x1 64->256 @1", 64, 1, 1, 256, 1, 1, 0, 1, "FDW", False),
    ("head0 3x3 128->256 @64", 128, 64, 64, 256, 3, 1, 1, 1, "FDW", True),
    ("head1 3x3 128->256 @128", 128, 128, 128, 256, 3, 1, 1, 1, "FDW", True),
    ("head2 3x3 256->64 @128", 256, 128, 128, 64, 3, 1, 1, 1, "FDW", True),
]
# fp32 classifiers (1x1 -> 19 with bias, logits at channel stride 32; dgrad through the 64-padded weight)
CLASSIFIERS = [("classifier 1x1 256->19 @64", 256, 64, 64), ("classifier 1x1 256->19 @128", 256, 128, 128),
               ("classifier 1x1 64->19 @128", 64, 128, 128)]

dev = torch.device("cuda:0")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def conv_case(C, H, W, K, R, st, pad, passes, stats):
    x = ops.nhwc_empty(N, C, H, W)
    x.normal_()
    wb = torch.randn(K, R, R, C, device=dev).to(torch.bfloat16)
    wt = torch.randn(C, R, R, K, device=dev).to(torch.bfloat16)
    P, Q = ops.conv_out_size(H, R, st, pad, 1), ops.conv_out_size(W, R, st, pad, 1)
    y = ops.nhwc_empty(N, K, P, Q)
    gy = ops.nhwc_empty(N, K, P, Q)
    gy.normal_()
    st_buf = torch.zeros(2, K, device=dev) if stats else None
    dw = torch.zeros(K, R, R, C, device=dev)
    dx = ops.nhwc_empty(N, C, H, W)
    fns = {"F": lambda: ops.conv_fprop(x, wb, K, R, st, pad, 1, out=y, stats=st_buf),
           "D": lambda: ops.conv_dgrad(gy, wt, (N, C, H, W), K, R, st, pad, 1, out=dx),
           "W": lambda: ops.conv_wgrad(x, gy, K, R, st, pad, 1, dw)}
    return 2.0 * N * P * Q * K * C * R * R, {p: timeit(fns[p]) for p in passes}


def classifier_case(C, H, W):
    K = 19
    x = ops.nhwc_empty(N, C, H, W)
    x.normal_()
    wb = torch.randn(K, 1, 1, C, device=dev).to(torch.bfloat16)
    wt = torch.randn(C, 1, 1, 64, device=dev).to(torch.bfloat16)
    bias = torch.randn(K, device=dev)
    y = ops.nhwc_empty(N, K, H, W, dtype=torch.float32, cs=32)
    gy = ops.nhwc_empty(N, 64, H, W)
    gy.normal_()
    dw = torch.zeros(K, 1, 1, C, device=dev)
    dx = ops.nhwc_empty(N, C, H, W)
    t = {"F": timeit(lambda: ops.conv_fprop(x, wb, K, 1, 1, 0, 1, bias=bias, out=y)),
         "D": timeit(lambda: ops.conv_dgrad(gy, wt, (N, C, H, W), 64, 1, 1, 0, 1, out=dx)),
         "W": timeit(lambda: ops.conv_wgrad(x, gy[:, :K], K, 1, 1, 0, 1, dw))}
    return 2.0 * N * H * W * K * C, t


def stem_pair():
    """the two 7x7/2 stems 3->64 @1024->512: two N = 64 fprop launches into one 128-channel buffer, one fused wgrad"""
    H = W = 1024
    xs = ops.pack_image_s2d(torch.randn(N, 3, H, W, device=dev))
    wp = torch.randn(128, 4, 4, 16, device=dev).to(torch.bfloat16)
    raw = ops.nhwc_empty(N, 128, H // 2, W // 2)
    stats = torch.zeros(2, 128, device=dev)
    gy = ops.nhwc_empty(N, 128, H // 2, W // 2)
    gy.normal_()
    dwp = torch.zeros(128, 4, 64, device=dev)

    def fprop():
        for off in (0, 64):
            ops.call("tsb_conv_stem_fprop", ops.ptr(xs), N, H, W, ops.ptr(wp[off:]), 64, ops.ptr(raw[:, off:]), 128,
                     ops.ptr(stats[0][off:]), ops.ptr(stats[1][off:]), *ops.det_ws(), ops.stream())

    def wgrad():
        ops.call("tsb_conv_stem_wgrad", ops.ptr(xs), N, H, W, ops.ptr(gy), 128, 128, ops.ptr(dwp), *ops.det_ws(), ops.stream())

    return 2.0 * N * (H // 2) * (W // 2) * 128 * 147, {"F": timeit(fprop), "W": timeit(wgrad)}


def main():
    args = sys.argv[1:]
    out_dir = None
    if "--out" in args:
        out_dir = args[args.index("--out") + 1]
    rows = []
    fl, t = stem_pair()
    rows.append(("stem pair 7x7/2 3->2x64 @1024", 1, fl, t))
    for name, C, H, W, K, R, st, pad, count, passes, stats in STEP:
        fl, t = conv_case(C, H, W, K, R, st, pad, passes, stats)
        rows.append((name, count, fl, t))
    for name, C, H, W in CLASSIFIERS:
        fl, t = classifier_case(C, H, W)
        rows.append((name, 1, fl, t))
    table = []
    total_us, total_fl = 0.0, 0.0
    print("%-34s %3s | %-17s | %-17s | %-17s" % ("shape", "x", "fprop us (TF/s)", "dgrad us (TF/s)", "wgrad us (TF/s)"))
    for name, count, fl, t in rows:
        cells = []
        for p in "FDW":
            if p in t:
                cells.append("%9.1f (%5.0f)" % (t[p], fl / t[p] / 1e6))
                total_us += count * t[p]
                total_fl += count * fl
                table.append({"shape": name, "count": count, "pass": {"F": "fprop", "D": "dgrad", "W": "wgrad"}[p],
                              "us": t[p], "tflops": fl / t[p] / 1e6, "gflop": fl / 1e9})
            else:
                cells.append("%17s" % "-")
        print("%-34s %3d | %s" % (name, count, " | ".join(cells)))
    print("step-weighted total: %.2f ms, %.0f TF/s (%.1f GFLOP)" % (total_us / 1e3, total_fl / total_us / 1e6, total_fl / 1e9))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_conv.json"), "w") as f:
            json.dump({"gpu": torch.cuda.get_device_name(0), "batch": N, "rows": table,
                       "step_ms": total_us / 1e3, "step_gflop": total_fl / 1e9}, f, indent=1)


if __name__ == "__main__":
    main()
