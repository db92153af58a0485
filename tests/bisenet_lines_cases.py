"""Seeded synthetic cases of the BiSeNet lines R18.speed, X39.speed and R101, shared by
tools/make_live_golden_bisenet_lines.py (live reference) and tests/test_cpu_bisenet_lines.py.

Same recipe as golden_cases.bisenet_case, generalised to non-square H x W images and labels at 1/gt_down resolution
(the .speed lines train against labels at 1/8, config.py gt_down_sampling = 8)."""
import torch


def bisenet_case(N, H, W, seed, gt_down=1):
    """H x W image and labels at 1/gt_down of it, the top tenth of the label rows ignored; min_kept as the reference
    train.py sets it, batch·H·W // (16·gt_down²)"""
    h, w = H // gt_down, W // gt_down
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, H, W, generator=g)
    y = torch.randint(0, 19, (N, h, w), generator=g, dtype=torch.int64)
    y[:, : h // 10, :] = 255
    return x, y, N * H * W // (16 * gt_down ** 2), seed
