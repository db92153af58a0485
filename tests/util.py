import torch


def rel_err(a, b):
    """max |a-b| / max|b| (scale-relative, robust for bf16 comparisons)"""
    a = a.detach().float().cpu()
    b = b.detach().float().cpu()
    denom = b.abs().max().clamp_min(1e-12)
    return float((a - b).abs().max() / denom)


def norm_err(a, b):
    a = a.detach().float().cpu()
    b = b.detach().float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


def bf16_round(t):
    return t.to(torch.bfloat16).to(torch.float32)


def make_labels(N, H, W, C, ignore, gen, ignore_frac=0.1):
    lab = torch.randint(0, C, (N, H, W), generator=gen, dtype=torch.int64)
    k = max(1, int(H * ignore_frac))
    lab[:, :k, :] = ignore  # deterministic ~10 % ignore band (SURVEY §8d)
    return lab


U24 = 2.0 ** -24   # unit roundoff of fp32


def lerp_matrix(n_in, n_out):
    """float64 [n_out, n_in] matrix of the fp32 bilinear weights (align_corners=True) that band.cuh make_lerp forms: row y
    holds l0 at i0 and l1 at i1 (summed when i0 == i1). Up-sampling is M_H @ x @ M_W^T, its adjoint M_H^T @ g @ M_W."""
    import numpy as np
    f = np.float32
    sc = f(n_in - 1) / f(n_out - 1) if n_out > 1 else f(0.0)
    src = sc * np.arange(n_out, dtype=f)
    i0 = np.minimum(src.astype(np.int64), n_in - 1)
    i1 = np.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = src - i0.astype(f)
    l0 = f(1.0) - l1
    M = np.zeros((n_out, n_in), dtype=np.float64)
    r = np.arange(n_out)
    np.add.at(M, (r, i0), l0.astype(np.float64))
    np.add.at(M, (r, i1), l1.astype(np.float64))
    return torch.from_numpy(M)


def band_extent(n_in, n_out):
    """largest number of output rows (columns) that share one left source row (column) i0: ny (nx / 2) of band_grad_k"""
    import numpy as np
    f = np.float32
    sc = f(n_in - 1) / f(n_out - 1) if n_out > 1 else f(0.0)
    i0 = np.minimum((sc * np.arange(n_out, dtype=f)).astype(np.int64), n_in - 1)
    return int(np.bincount(i0).max())


def band_grad_k(M, C, ny, nx):
    """K of the per-element bound |got - ref| <= K * 2^-24 * A of the up-sampled loss gradients (derivation:
    test_gpu_loss_exact.py). M = max |low-res logit|, C classes, ny rows per band, nx columns per low-res column pair."""
    return 17 * M + 2 * C + ny + nx + ny * nx + 34
