"""Kernel times of the stem region of the BiSeNet-R18 training step (StemPairFn at 16 x 1024^2: the 128-channel
stem map [N,128,512,512], spatial half = channels 0..63, context half = channels 64..127 → 3x3/2 max pool).

    python tools/bench_stem.py [--batch 16] [--size 1024] [--iters 50] [--out DIR]

Each libtsb entry point of the stem's BatchNorm / ReLU / max-pool passes is timed with CUDA events over --iters
back-to-back launches on seeded inputs, with its algorithmic HBM bytes (each operand read or written once, from the
shapes), the achieved GB/s and that rate's share of the H100 SXM data-sheet 3.35 TB/s, for both ways of running the
forward (the backward is the same in both: tsb_maxpool3x3s2_bwd on the context half, then tsb_bn_bwd_reduce /
tsb_bn_bwd_apply on each half):
  unfused: tsb_bn_apply over all 128 channels, then tsb_maxpool3x3s2_fwd on the context half;
  fused:   tsb_bn_apply on the spatial half and tsb_bn_apply_maxpool3x3s2 on the context half.
Prints one JSON line (also written to DIR/bench_stem.json) with the card name, power limit and max SM clock read in
the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e)[:200])


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_stem.py times kernels on the GPU"
    from torchseg_b200 import ops
    from torchseg_b200.ops import call, ptr, det_ws, stream
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    N = args.batch
    P = Q = args.size // 2                # stem map (7x7/2 conv output)
    P2, Q2 = (P - 1) // 2 + 1, (Q - 1) // 2 + 1   # after the 3x3/2 max pool
    K, K1 = 128, 64
    K2 = K - K1
    npix = N * P * Q
    g = torch.Generator(device=dev).manual_seed(0)
    raw = ops.nhwc_empty(N, K, P, Q, device=dev)
    raw.copy_(torch.randn(raw.shape, generator=g, device=dev))
    gamma = torch.rand(K, generator=g, device=dev) + 0.5
    beta = torch.randn(K, generator=g, device=dev) * 0.1
    mean = torch.randn(K, generator=g, device=dev) * 0.1
    invstd = torch.rand(K, generator=g, device=dev) + 0.5
    aux = torch.stack([mean, invstd, gamma * invstd, beta - mean * gamma * invstd]).contiguous()
    y = ops.nhwc_empty(N, K, P, Q, device=dev)
    pool = ops.nhwc_empty(N, K2, P2, Q2, device=dev)
    idx = torch.empty((N, P2, Q2, K2), dtype=torch.uint8, device=dev)
    dpool = ops.nhwc_empty(N, K2, P2, Q2, device=dev)
    dpool.copy_(torch.randn(dpool.shape, generator=g, device=dev))
    dy_sp = ops.nhwc_empty(N, K1, P, Q, device=dev)
    dy_sp.copy_(torch.randn(dy_sp.shape, generator=g, device=dev))
    dy_ctx = ops.nhwc_empty(N, K2, P, Q, device=dev)
    draw = ops.nhwc_empty(N, K, P, Q, device=dev)
    red = torch.zeros((2, K), dtype=torch.float32, device=dev)
    count = float(npix)
    B = 2   # bytes per bf16 element
    big = npix * B             # bytes per channel of the stem map
    small = N * P2 * Q2        # elements per channel of the pooled map (bf16 value + uint8 argmax each)

    def bwd_reduce(h, dy, Kh):
        call("tsb_bn_bwd_reduce", ptr(dy), ops.cs_of(dy), None, 0, ptr(raw[:, h]), K, ptr(aux[0, h]), ptr(aux[1, h]), 1,
             npix, Kh, ptr(red[0, h]), ptr(red[1, h]), ptr(aux[2, h]), ptr(aux[3, h]), *det_ws(), stream())

    def bwd_apply(h, dy, Kh):
        call("tsb_bn_bwd_apply", ptr(dy), ops.cs_of(dy), None, 0, ptr(raw[:, h]), K, ptr(aux[0, h]), ptr(aux[1, h]),
             ptr(gamma[h]), ptr(red[0, h]), ptr(red[1, h]), count, 1, ptr(draw[:, h]), K, None, 0, npix, Kh, None, None,
             ptr(aux[2, h]), ptr(aux[3, h]), stream())

    sp, cx = slice(0, K1), slice(K1, K)
    pooled = K2 * small * (B + 1)   # pooled map + argmax
    launches = [
        # (name, fn, algorithmic bytes)
        ("tsb_bn_apply (128 ch)", lambda: call("tsb_bn_apply", ptr(raw), K, ptr(aux[2]), ptr(aux[3]), None, 0, 1, ptr(y),
                                               K, npix, K, stream()), 2 * K * big),
        ("tsb_maxpool3x3s2_fwd (context half)", lambda: call("tsb_maxpool3x3s2_fwd", ptr(y[:, cx]), K, ptr(pool), K2,
                                                             ptr(idx), N, K2, P, Q, stream()),
         K2 * big + K2 * small * (B + 1)),
        ("tsb_maxpool3x3s2_bwd (context half)", lambda: call("tsb_maxpool3x3s2_bwd", ptr(idx), ptr(dpool), K2,
                                                             ptr(dy_ctx), K2, N, K2, P, Q, stream()),
         K2 * small * (B + 1) + K2 * big),
        ("tsb_bn_bwd_reduce (spatial half)", lambda: bwd_reduce(sp, dy_sp, K1), 2 * K1 * big),
        ("tsb_bn_bwd_reduce (context half)", lambda: bwd_reduce(cx, dy_ctx, K2), 2 * K2 * big),
        ("tsb_bn_bwd_apply (spatial half)", lambda: bwd_apply(sp, dy_sp, K1), 3 * K1 * big),
        ("tsb_bn_bwd_apply (context half)", lambda: bwd_apply(cx, dy_ctx, K2), 3 * K2 * big),
        ("tsb_bn_apply (spatial half)", lambda: call("tsb_bn_apply", ptr(raw), K, ptr(aux[2]), ptr(aux[3]), None, 0, 1,
                                                     ptr(y), K1, npix, K1, stream()), 2 * K1 * big),
        ("tsb_bn_apply_maxpool3x3s2 (context half)",
         lambda: call("tsb_bn_apply_maxpool3x3s2", ptr(raw[:, cx]), K, ptr(aux[2, cx]), ptr(aux[3, cx]), ptr(pool), K2,
                      ptr(idx), N, K2, P, Q, stream()), K2 * big + pooled),
    ]
    unfused = ["tsb_bn_apply (128 ch)", "tsb_maxpool3x3s2_fwd (context half)", "tsb_maxpool3x3s2_bwd (context half)",
               "tsb_bn_bwd_reduce (spatial half)", "tsb_bn_bwd_reduce (context half)",
               "tsb_bn_bwd_apply (spatial half)", "tsb_bn_bwd_apply (context half)"]
    fused = ["tsb_bn_apply (spatial half)", "tsb_bn_apply_maxpool3x3s2 (context half)"] + unfused[2:]
    rows = {}
    for name, fn, nbytes in launches:
        ms = time_ms(fn, args.iters)
        rows[name] = dict(launch=name, ms=round(ms, 4), bytes=nbytes, gbs=round(nbytes / ms / 1e6, 1),
                          share_of_3350=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))

    def total(names):
        return dict(ms=round(sum(rows[n]["ms"] for n in names), 4), bytes=sum(rows[n]["bytes"] for n in names))

    line = dict(tool="bench_stem", batch=N, stem_map=[N, K, P, Q], iters=args.iters, gpu=gpu_info(),
                launches=list(rows.values()), unfused=total(unfused), fused=total(fused))
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_stem.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
