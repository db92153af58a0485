"""The stem's fused BatchNorm-apply + ReLU + 3x3/2 max-pool pass against the unfused kernel pair, bit for bit.

tsb_bn_apply_maxpool3x3s2 must give the pooled map and argmax of tsb_bn_apply (ReLU) → tsb_maxpool3x3s2_fwd. The raw
map is a channel slice of a wider buffer whose other channels hold NaN, as the context half of the 128-channel stem
map is; cases cover odd map sizes (padded last row and column), ties and all-negative windows (integer inputs, channels
whose shift drives every value below zero), channel counts on both sides of the hoisted-parameter path, and a batch
that takes several trips of the grid. A profiled BiSeNet-R18 step must run the fused pass and not maxpool_fwd_kernel;
BiSeNet-X39, whose stem is not fused, still runs maxpool_fwd_kernel."""
import re

import pytest
import torch

from util import make_labels

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SENT = 0x7FA5   # bf16 NaN bit pattern no kernel computes

# (N, C, H, W, channel stride of raw, channel offset of the slice, integer inputs)
CASES = [
    (2, 64, 57, 75, 128, 64, True),     # the stem's context half of an odd image: ties, padded last row and column
    (2, 64, 58, 76, 128, 64, False),    # even map, real-valued inputs
    (3, 24, 9, 7, 40, 8, True),         # C8 = 3 does not divide the CTA: per-vector parameter loads
    (1, 8, 1, 1, 8, 0, True),           # a single pixel
    (2, 16, 1, 6, 32, 16, False),       # one row
    (40, 64, 96, 96, 128, 64, True),    # several trips of every grid
]


def _bits(t):
    return t.contiguous().view(torch.int16)


def _call(name, *args):
    from torchseg_b200 import ops
    ops.call(name, *args, ops.stream())


def _params(C, g):
    """per-channel scale, shift (fp32, 16-byte aligned) of a BatchNorm; one channel in four is shifted so far below
    zero that its ReLU output is all zero"""
    mean = torch.randn(C, generator=g, device="cuda") * 0.5
    invstd = torch.rand(C, generator=g, device="cuda") + 0.5
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    beta = torch.randn(C, generator=g, device="cuda") * 0.5
    scale = gamma * invstd
    shift = beta - mean * scale
    shift[::4] = -1e3
    return scale.contiguous(), shift.contiguous()


@pytest.mark.parametrize("case", CASES, ids=["N%dC%dH%dW%dcs%d@%d%s" % (c[:6] + ("int" if c[6] else "",)) for c in CASES])
def test_fused_stem_pool_matches_unfused(cuda, case):
    N, C, H, W, cs, off, ints = case
    P, Q = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    npix = N * H * W
    g = torch.Generator(device="cuda").manual_seed(N * 1000 + C * 10 + H)
    buf = torch.full((N, H, W, cs), float("nan"), dtype=BF, device="cuda")
    if ints:   # small integers: many ties inside each window after the affine map and the bf16 rounding
        buf[..., off:off + C] = torch.randint(-3, 4, (N, H, W, C), generator=g, device="cuda").to(BF)
    else:
        buf[..., off:off + C] = torch.randn((N, H, W, C), generator=g, device="cuda").to(BF)
    x = buf[..., off:]
    scale, shift = _params(C, g)

    # forward: the unfused pair ...
    y = torch.empty((N, H, W, C), dtype=BF, device="cuda")
    _call("tsb_bn_apply", x.data_ptr(), cs, scale.data_ptr(), shift.data_ptr(), None, 0, 1, y.data_ptr(), C, npix, C)
    pool_ref = torch.empty((N, P, Q, C), dtype=BF, device="cuda")
    am_ref = torch.empty((N, P, Q, C), dtype=torch.uint8, device="cuda")
    _call("tsb_maxpool3x3s2_fwd", y.data_ptr(), C, pool_ref.data_ptr(), C, am_ref.data_ptr(), N, C, H, W)
    # ... and the fused pass, into a wider output whose pad channels must keep their bits
    pool = torch.full((N, P, Q, C + 8), SENT, dtype=torch.int16, device="cuda").view(BF)
    am = torch.full((N, P, Q, C), 255, dtype=torch.uint8, device="cuda")
    _call("tsb_bn_apply_maxpool3x3s2", x.data_ptr(), cs, scale.data_ptr(), shift.data_ptr(), pool.data_ptr(), C + 8,
          am.data_ptr(), N, C, H, W)
    assert torch.equal(_bits(pool[..., :C]), _bits(pool_ref)), "pooled map differs from bn_apply → maxpool_fwd"
    assert torch.equal(am, am_ref), "argmax differs from bn_apply → maxpool_fwd"
    assert bool((_bits(pool[..., C:]) == SENT).all()), "the fused forward wrote a pad channel"
    if ints:
        assert bool((pool_ref == 0).any()), "the case has no all-negative window"


_UNFUSED = re.compile(r"(?<![A-Za-z0-9_])maxpool_fwd_kernel")
_FUSED = re.compile(r"bn_relu_maxpool_fwd_kernel")


def _step_kernels(model, x, y):
    """names of the kernels one training step (forward + backward) launches"""
    from torch.profiler import ProfilerActivity, profile
    model(x, y).backward()   # warm-up: packs, workspaces
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(x, y).backward()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


def test_r18_step_runs_the_fused_stem_and_x39_the_unfused_pool(cuda):
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.networks.bisenet_x39 import BiSeNet as BiSeNetX39
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    N, H, W = 2, 128, 160
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, 3, H, W, generator=g).to(cuda)
    y = make_labels(N, H, W, 19, 255, g).to(cuda)
    ohem = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=N * H * W // 16, use_weight=False)
    torch.manual_seed(0)
    r18 = torchseg_b200.prepare_model(BiSeNet(19, True, ohem, None, torch.nn.BatchNorm2d).to(cuda))
    r18.train()
    names = _step_kernels(r18, x, y)
    assert not [n for n in names if _UNFUSED.search(n)], "the R18 step still runs maxpool_fwd_kernel"
    assert len([n for n in names if _FUSED.search(n)]) == 1, "the R18 step should run the fused stem pass once"

    x39 = BiSeNetX39(19, True, torch.nn.CrossEntropyLoss(ignore_index=255), ohem, None, torch.nn.BatchNorm2d)
    x39 = torchseg_b200.prepare_model(x39.to(cuda))
    x39.train()
    names = _step_kernels(x39, x, y)
    assert [n for n in names if _UNFUSED.search(n)], "X39 should still run maxpool_fwd_kernel"
    assert not [n for n in names if _FUSED.search(n)]
