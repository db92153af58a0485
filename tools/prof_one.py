"""a handful of launches of the hot kernels at BASELINE size for `ncu --set full` (keep it short: ncu replays ~40x)
   ncu --set full --clock-control none --import-source on -k regex:'igemm|wgrad|ohem' -s <skip> -c <n> -o prof python tools/prof_one.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torchseg_b200 import ops
dev = torch.device("cuda:0")
N, C, H, W, K = 16, 64, 256, 256, 64
x = ops.nhwc_empty(N, C, H, W); x.normal_()
wb = torch.randn(K, 3, 3, C, device=dev).to(torch.bfloat16)
y = ops.nhwc_empty(N, K, H, W); gy = ops.nhwc_empty(N, K, H, W); gy.normal_()
stats = torch.zeros(2, K, device=dev); dw = torch.zeros(K, 3, 3, C, device=dev)
x2 = ops.nhwc_empty(N, 128, 128, 128); x2.normal_()
wb2 = torch.randn(128, 3, 3, 128, device=dev).to(torch.bfloat16)
y2 = ops.nhwc_empty(N, 128, 128, 128); st2 = torch.zeros(2, 128, device=dev)
gy2 = ops.nhwc_empty(N, 128, 128, 128); gy2.normal_(); dw2 = torch.zeros(128, 3, 3, 128, device=dev)
# OHEM head (x8): low-res fp32 NHWC logits, channel stride 32
g = torch.Generator().manual_seed(0)
lo = ops.nhwc_zeros(N, 19, 128, 128, dtype=torch.float32, device=dev, cs=32)
lo.copy_(torch.randn(N, 19, 128, 128, generator=g).to(dev))
labels = torch.randint(0, 19, (N, 1024, 1024), generator=g).to(dev)
labels[:, :102] = 255
for _ in range(2):
    ops.conv_fprop(x, wb, K, 3, 1, 1, 1, out=y, stats=stats)         # layer1 64->64 @256 (BN=64, resident weights, row tiles)
    ops.conv_fprop(x2, wb2, 128, 3, 1, 1, 1, out=y2, stats=st2)      # layer2 128->128 @128 (BN=128, streamed weights, pairs)
    ops.conv_wgrad(x, gy, K, 3, 1, 1, 1, dw)                          # layer1 wgrad (nine-tap kernel)
    ops.conv_wgrad(x2, gy2, 128, 3, 1, 1, 1, dw2)                     # layer2 wgrad (nine-tap kernel)
    lo_ = lo.detach().requires_grad_(True)
    loss = ops.OhemUpCEFn.apply(lo_, labels, 1024, 1024, 19, 255, 0.7, N * 1024 * 1024 // 16, None)
    loss.backward()
torch.cuda.synchronize()
print("ok")
