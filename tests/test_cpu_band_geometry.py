"""A float32 model of the band geometry of the fused up-sampling loss kernels (torchseg_b200/csrc/band.cuh) and of the host
dispatch of tsb_ohem_ptarget_up / tsb_ohem_grad_up (ohem.cu) and tsb_ce_up_fwd / tsb_ce_up_bwd (ce_up.cu), swept over the
model shapes and a few thousand seeded random geometries.

Every formula is written with numpy float32 scalars in the device's operation order, next to the band.cuh line it
restates, so that a change to either shows up in review. Checked:
1. each hi-res row y belongs to exactly one band, ci = make_lerp(ry, y, h).i0, and lies in that band's [y_lo, y_hi];
2. ncols <= band_maxcols for every strip;
3. the segment walk of col_sums sends each strip column's l0 weight to exactly lx.i0 and its l1 weight to exactly lx.i1,
   once each, including the clamped last column and the low-res columns a down-scale skips;
4. whenever the host picks ohem_grad_up_x_kernel, the bands of one of its four launches write disjoint low-res cells;
5. every geometry is accepted by both halves of a forward / backward pair, or refused by the forward;
and that the model shapes keep the kernels they ran before those two checks existed.
The last test runs an fp32 emulation of the band backward against the per-element bound of test_gpu_loss_exact.py, and
three wrong walks that it must reject.
"""
import numpy as np
import pytest
import torch

from util import U24, band_extent, band_grad_k, lerp_matrix

f32 = np.float32
OHEM_STRIP, CE_STRIP = 256, 64
OHEM_PITCH, CE_TQ = OHEM_STRIP + 1, (CE_STRIP + 1) * 4

# (h, H, w, W): the networks' low-res logits → label resolution
MODEL_SHAPES = [
    (128, 1024, 128, 1024),   # x8: BiSeNet main and aux at /8, FCN, DFN border
    (64, 1024, 64, 1024),     # x16: BiSeNet aux at /16
    (32, 1024, 32, 1024),     # x32: DFN
    (16, 512, 16, 512),       # x32: DFN at 512
    (128, 1024, 256, 2048),   # x8 at the Cityscapes full frame
    (64, 1024, 128, 2048),    # x16 at the full frame
    (90, 713, 90, 713),       # PSPNet
    (60, 473, 60, 473),       # PSANet
    (64, 512, 64, 512),       # x8 at 512 (VOC)
]


# ------------------------------------------------------------------------------------------------ band.cuh, in float32
def area_scale(n_in, n_out):                          # band.cuh:41-43
    return f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0.0)


def make_lerp(scale, dst, n_in):                      # band.cuh:22-31 (dst may be an int array)
    src = f32(scale) * np.asarray(dst).astype(f32)    # :24 __fmul_rn(scale, (float)dst)
    i0 = np.minimum(src.astype(np.int64), n_in - 1)   # :25-26 truncation, clamp
    i1 = i0 + (i0 < n_in - 1)                         # :27
    l1 = (src - i0.astype(f32)).astype(f32)           # :28
    l0 = (f32(1.0) - l1).astype(f32)                  # :29
    return i0, i1, l0, l1


def band_geom(ry, rx, ci, x0, x1, h, H, w):           # band.cuh:50-62
    i1 = ci + (1 if ci < h - 1 else 0)                # :53
    if ry > 0:
        y_lo = max(0, int(np.floor(f32(ci) / ry)) - 1)              # :55
        y_hi = min(H - 1, int(np.ceil(f32(ci + 1) / ry)) + 1)       # :56
    else:
        y_lo, y_hi = 0, H - 1                         # :57
    a0 = int(make_lerp(rx, x0, w)[0])                 # :58
    b1 = int(make_lerp(rx, x1 - 1, w)[1])
    return i1, y_lo, y_hi, a0, b1 - a0 + 1            # :59-60 jbase, ncols


def band_maxcols(strip, w, W):                        # band.cuh:64
    return (strip * w + W - 1) // W + 3


def seg_table(rx, x0, x1, w, jbase, ncols):
    """seg_init / seg_fill (band.cuh:99-114): s_seg, s_l0, s_l1 of one strip"""
    nx = x1 - x0
    seg = [nx] * (ncols + 2)                          # :106
    x = np.arange(x0, x1)
    i0, _, l0, l1 = make_lerp(rx, x, w)               # :103-104 (every column of the strip is inside the image)
    for col in range(nx):                             # :108-113, one owner per column
        jprev = -1 if col == 0 else int(i0[col - 1]) - jbase          # :111 make_lerp(rx, x - 1, w).i0
        for jj in range(jprev + 1, int(i0[col]) - jbase + 1):
            seg[jj] = col
    return seg, l0, l1


def col_walk(seg, s_l0, s_l1, jbase, ncols, w, mutant=None):
    """the column walk of col_sums (band.cuh:121-146): for each low-res column j the list of (strip column, weight) it
    sums, in order. `mutant` replaces the walk by a wrong one (the bound test must reject it)."""
    out = []
    for j in range(ncols):
        a0, a1 = seg[j], seg[j + 1]                   # :124
        terms = [(xx, s_l0[xx]) for xx in range(a0, a1)]               # :125-129
        clamped = jbase + j == w - 1                  # :130
        b0 = a0 if clamped else (seg[j - 1] if j > 0 else 0)           # :131
        b1 = a1 if clamped else (a0 if j > 0 else 0)                   # :132
        wr = s_l0 if (clamped and mutant == "swap_clamped") else s_l1
        terms += [(xx, wr[xx]) for xx in range(b0, b1)]                # :133-137
        if clamped and j > 0:                                          # :138-144
            terms += [(xx, wr[xx]) for xx in range(seg[j - 1], a0)]
        out.append(terms)
    return out


# ------------------------------------------------------------------------------------------------ host dispatch
def strips_disjoint(w, W, strip=OHEM_STRIP):
    """ohem.cu same_parity_strips_disjoint"""
    rx = area_scale(w, W)
    s = 0
    while (s + 2) * strip < W:
        il = min(int(f32(rx) * f32((s + 1) * strip - 1)), w - 1)
        i_first = min(int(f32(rx) * f32((s + 2) * strip)), w - 1)
        if il + (1 if il < w - 1 else 0) >= i_first:
            return False
        s += 1
    return True


def ohem_grad_up_path(C, w, W, exact_rule=True):
    """ohem.cu grad_up_path: None (refused), "x" (ohem_grad_up_x_kernel) or "generic". exact_rule=False is the rule
    before the strip check: shared memory alone."""
    maxcols = band_maxcols(OHEM_STRIP, w, W)
    if C < 1 or C > 32 or maxcols > OHEM_STRIP:
        return None
    if C in (19, 21):
        smx = 4 * (2 * C * OHEM_PITCH + 2 * maxcols * C)
        if smx <= 72 * 1024 and (not exact_rule or strips_disjoint(w, W)):
            return "x"
    cmax = 20 if C <= 20 else 32
    return "generic" if 4 * (2 * cmax * OHEM_PITCH + 2 * maxcols * cmax) <= 96 * 1024 else None


def ohem_ptarget_up_path(C, w, W, check_backward=True):
    """tsb_ohem_ptarget_up; check_backward=False is the rule before it refused what the backward refuses"""
    if C < 1 or C > 32 or (check_backward and ohem_grad_up_path(C, w, W) is None):
        return None
    maxcols = band_maxcols(OHEM_STRIP, w, W)
    if C in (19, 21) and 4 * (2 * C * OHEM_PITCH + 2 * maxcols * C) <= 100 * 1024:
        return "x"
    cmax = 20 if C <= 20 else 32
    return "generic" if 4 * 2 * maxcols * cmax <= 28 * 1024 else None


def ce_up_bwd_ok(C, w, W):
    """ce_up.cu bwd_smem != 0"""
    maxcols = band_maxcols(CE_STRIP, w, W)
    return 1 <= C <= 152 and maxcols <= CE_STRIP and 4 * (2 * ((C + 3) // 4) * CE_TQ + 4 * maxcols * C) <= 110 * 1024


def ce_up_fwd_ok(C, w, W, check_backward=True):
    maxcols = band_maxcols(CE_STRIP, w, W)
    ok = 1 <= C <= 152 and 4 * (2 * ((C + 3) // 4) * CE_TQ + 2 * maxcols * C) <= 110 * 1024
    return ok and (not check_backward or ce_up_bwd_ok(C, w, W))


# ------------------------------------------------------------------------------------------------ geometries
def _random_geometries(n=3000, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        kind = rng.integers(0, 8)
        h, w = int(rng.integers(1, 160)), int(rng.integers(1, 160))
        if kind == 0:      # non-integer up-scale
            H, W = int(h * rng.uniform(1, 12)) + 1, int(w * rng.uniform(1, 12)) + 1
        elif kind == 1:    # one of each extent
            h, H, w, W = [int(v) for v in rng.choice([1, 2, 3, 7], 4)]
            H, W = H * int(rng.integers(1, 40)), W * int(rng.integers(1, 40))
        elif kind == 2:    # W = k * strip + 1
            W = int(rng.choice([OHEM_STRIP, CE_STRIP])) * int(rng.integers(1, 9)) + 1
            H = int(rng.integers(1, 1200))
        elif kind == 3:    # W smaller than one strip
            W, H = int(rng.integers(1, 64)), int(rng.integers(1, 600))
        elif kind == 4:    # very large scale (w, h small, W, H large)
            h, w = int(rng.integers(1, 5)), int(rng.integers(1, 5))
            H, W = int(rng.integers(100, 2500)), int(rng.integers(100, 2500))
        elif kind == 5:    # down-scale and near-identity
            H, W = max(1, int(h * rng.uniform(0.3, 1.1))), max(1, int(w * rng.uniform(0.3, 1.1)))
        elif kind == 6:    # integer scales
            s = int(rng.choice([2, 4, 8, 16, 32]))
            H, W = h * s, w * s
        else:              # align-corners-exact scales (n - 1) * s + 1
            s = int(rng.integers(2, 40))
            H, W = (h - 1) * s + 1, (w - 1) * s + 1
        out.append((h, H, w, W))
    return out


RANDOM = _random_geometries()
EXTRA = [(1, 1, 1, 1), (1, 7, 1, 9), (5, 1, 6, 1), (4, 4, 300, 300), (2, 600, 2, 600), (3, 3, 2, 600)]
ALL = MODEL_SHAPES + EXTRA + RANDOM


def _strips(W, strip):
    return [(x0, min(W, x0 + strip)) for x0 in range(0, W, strip)]


# ------------------------------------------------------------------------------------------------ 1. and 2.
def test_rows_belong_to_one_band():
    for h, H, w, W in ALL:
        ry = area_scale(h, H)
        y = np.arange(H)
        ci = make_lerp(ry, y, h)[0]
        assert ci.min() >= 0 and ci.max() <= h - 1
        lo_hi = np.array([band_geom(ry, f32(0), c, 0, 1, h, H, w)[1:3] for c in range(h)])
        assert np.all(lo_hi[ci, 0] <= y) and np.all(y <= lo_hi[ci, 1]), (h, H, w, W)


@pytest.mark.parametrize("strip", [OHEM_STRIP, CE_STRIP])
def test_ncols_within_maxcols(strip):
    for h, H, w, W in ALL:
        rx = area_scale(w, W)
        x0 = np.arange(0, W, strip)
        x1 = np.minimum(W, x0 + strip)
        ncols = make_lerp(rx, x1 - 1, w)[1] - make_lerp(rx, x0, w)[0] + 1
        assert ncols.max() <= band_maxcols(strip, w, W), (h, H, w, W, strip)


# ------------------------------------------------------------------------------------------------ 3.
def _check_walk_weights(w, W, strip):
    """walk with the weights tagged (l0 -> 1, l1 -> 2): column x's tags must arrive at i0 and i1 once each, on the first,
    a middle and the last strip"""
    rx = area_scale(w, W)
    strips = _strips(W, strip)
    for x0, x1 in sorted({strips[0], strips[len(strips) // 2], strips[-1]}):
        _, _, _, jbase, ncols = band_geom(f32(0), rx, 0, x0, x1, 1, 1, w)
        seg, _, _ = seg_table(rx, x0, x1, w, jbase, ncols)
        nx = x1 - x0
        tag0, tag2 = np.ones(nx), np.full(nx, 2.0)
        i0, i1, _, _ = make_lerp(rx, np.arange(x0, x1), w)
        got = np.zeros((nx, ncols))
        for j, terms in enumerate(col_walk(seg, tag0, tag2, jbase, ncols, w)):
            for xx, t in terms:
                got[xx, j] += t
        want = np.zeros((nx, ncols))
        np.add.at(want, (np.arange(nx), i0 - jbase), 1.0)
        np.add.at(want, (np.arange(nx), i1 - jbase), 2.0)
        assert np.array_equal(got, want), (w, W, strip, x0)


@pytest.mark.parametrize("strip", [OHEM_STRIP, CE_STRIP])
def test_column_walk_routes_every_weight_once(strip):
    for h, H, w, W in ALL[:1200]:
        _check_walk_weights(w, W, strip)


# ------------------------------------------------------------------------------------------------ 4. and 5.
def _x_launch_cells_disjoint(h, w, W):
    """ohem_grad_up_x_kernel launch `ph` runs bands (ci, s) with ci % 2 == ph & 1 and s % 2 == ph >> 1; band (ci, s)
    may write rows {ci, i1} x columns [jbase, jbase + ncols) of the low-res gradient. Rows and columns factor, so the
    cells of one launch are disjoint iff no row and no column is claimed twice."""
    rx = area_scale(w, W)
    strips = _strips(W, OHEM_STRIP)
    for ph in range(4):
        rows = np.zeros(h, dtype=np.int64)
        for ci in range(ph & 1, h, 2):
            for r in {ci, ci + (1 if ci < h - 1 else 0)}:
                rows[r] += 1
        cols = np.zeros(w, dtype=np.int64)
        for s in range(ph >> 1, len(strips), 2):
            x0, x1 = strips[s]
            _, _, _, jbase, ncols = band_geom(f32(0), rx, 0, x0, x1, 1, 1, w)
            cols[jbase:jbase + ncols] += 1
        if rows.max() > 1 or cols.max() > 1:
            return False
    return True


def test_exact_gradient_kernel_launches_write_disjoint_cells():
    for h, H, w, W in ALL:
        for C in (19, 21):
            if ohem_grad_up_path(C, w, W) == "x":
                assert _x_launch_cells_disjoint(h, w, W), (C, h, H, w, W)


def test_the_strip_rule_is_needed():
    """w = 2, W = 600, C = 19: shared memory alone picks the exact-class kernel, whose strips 0 and 2 both write low-res
    columns {0, 1} in one launch; the strip rule sends it to the generic kernel"""
    assert ohem_grad_up_path(19, 2, 600, exact_rule=False) == "x"
    assert not _x_launch_cells_disjoint(2, 2, 600)
    assert ohem_grad_up_path(19, 2, 600) == "generic"


OHEM_CS = list(range(1, 33))
CE_CS = [1, 2, 5, 19, 32, 33, 64, 100, 149, 150, 151, 152]


def test_forward_accepts_only_what_the_backward_runs():
    for h, H, w, W in ALL:
        for C in OHEM_CS:
            if ohem_ptarget_up_path(C, w, W) is not None:
                assert ohem_grad_up_path(C, w, W) is not None, ("ohem", C, h, H, w, W)
        for C in CE_CS:
            if ce_up_fwd_ok(C, w, W):
                assert ce_up_bwd_ok(C, w, W), ("ce_up", C, h, H, w, W)


def test_forward_refusals_are_needed():
    """without the backward's rule, the forward accepts C = 19 at H = h, W = w and a 150-class head at x4, which the
    backward then refuses"""
    assert ohem_ptarget_up_path(19, 300, 300, check_backward=False) == "x"
    assert ohem_grad_up_path(19, 300, 300) is None and ohem_ptarget_up_path(19, 300, 300) is None
    assert ce_up_fwd_ok(150, 64, 256, check_backward=False)
    assert not ce_up_bwd_ok(150, 64, 256) and not ce_up_fwd_ok(150, 64, 256)


def test_model_shapes_keep_their_kernels():
    for h, H, w, W in MODEL_SHAPES:
        for C in OHEM_CS:
            assert ohem_grad_up_path(C, w, W) == ohem_grad_up_path(C, w, W, exact_rule=False)
            assert ohem_ptarget_up_path(C, w, W) == ohem_ptarget_up_path(C, w, W, check_backward=False)
        for C in (19, 21):
            assert ohem_grad_up_path(C, w, W) == "x" and ohem_ptarget_up_path(C, w, W) == "x"
        assert ce_up_fwd_ok(150, w, W) and ce_up_bwd_ok(150, w, W)


# ------------------------------------------------------------------------------------------------ the bound has teeth
def _fma32(a, b, c):
    return f32(np.float64(a) * np.float64(b) + np.float64(c))


def _emulate_grad(lo, labels, strip, mutant=None):
    """fp32 emulation of the band backward (ohem_grad_up_kernel / ce_up_bwd_kernel) of mean cross-entropy without
    ignored pixels: per band, G0 / G1 = fmaf over the member rows of l0y / l1y * (softmax - onehot) / count (in the
    kernel's blend order), then the col_sums walk into the low-res gradient. lo: float32 [C, h, w]."""
    C, h, w = lo.shape
    H, W = labels.shape
    ry, rx = area_scale(h, H), area_scale(w, W)
    wt = f32(1.0) / f32(H * W)
    d = np.zeros((C, h, w), dtype=f32)
    for x0, x1 in _strips(W, strip):
        _, _, _, jbase, ncols = band_geom(f32(0), rx, 0, x0, x1, 1, 1, w)
        seg, s_l0, s_l1 = seg_table(rx, x0, x1, w, jbase, ncols)
        walk = col_walk(seg, s_l0, s_l1, jbase, ncols, w, mutant)
        if mutant == "drop_edge":
            # the smallest weight a strip-edge column delivers, among those of at least 2^-8: the clamped last image
            # column's l1 is 0 up to one rounding of make_lerp, and dropping a term that small is rounding
            edge = [(j, k) for j, t in enumerate(walk) for k, (xx, wgt) in enumerate(t)
                    if xx in (0, x1 - x0 - 1) and wgt >= 2.0 ** -8]
            j, k = min(edge, key=lambda e: walk[e[0]][e[1]][1])
            del walk[j][k]
        i0x, i1x, l0x, l1x = make_lerp(rx, np.arange(x0, x1), w)
        for ci in range(h):
            i1, y_lo, y_hi, _, _ = band_geom(ry, rx, ci, x0, x1, h, H, w)
            rows = [y for y in range(y_lo, y_hi + 1) if make_lerp(ry, y, h)[0] == ci]
            if mutant == "drop_last_row":
                rows = rows[:-1]
            t0 = (l0x * lo[:, ci, i0x] + l1x * lo[:, ci, i1x]).astype(f32)       # lerp_h, [C, nx]
            t1 = (l0x * lo[:, i1, i0x] + l1x * lo[:, i1, i1x]).astype(f32)
            G0 = np.zeros_like(t0)
            G1 = np.zeros_like(t0)
            for y in rows:
                _, _, l0y, l1y = make_lerp(ry, y, h)
                v = (l0y * t0 + l1y * t1).astype(f32)                             # lerp_v
                e = np.exp(v - v.max(axis=0)).astype(f32)
                gg = (e * (wt / e.sum(axis=0, dtype=f32))).astype(f32)
                gg[labels[y, x0:x1], np.arange(x1 - x0)] -= wt
                G0 = (np.float64(l0y) * gg + G0).astype(f32)                      # fmaf
                G1 = (np.float64(l1y) * gg + G1).astype(f32)
            for j, terms in enumerate(walk):
                top, bot = np.zeros(C, dtype=f32), np.zeros(C, dtype=f32)
                for xx, wgt in terms:
                    top = (np.float64(wgt) * G0[:, xx] + top).astype(f32)
                    bot = (np.float64(wgt) * G1[:, xx] + bot).astype(f32)
                d[:, ci, jbase + j] += top
                d[:, i1, jbase + j] += bot
    return d


def _reference_and_bound(lo, labels):
    C, h, w = lo.shape
    H, W = labels.shape
    Mh, Mw = lerp_matrix(h, H), lerp_matrix(w, W)
    up = torch.einsum("Yh,chw,Xw->cYX", Mh, torch.from_numpy(lo).double(), Mw)
    p = torch.softmax(up, dim=0)
    oh = torch.nn.functional.one_hot(torch.from_numpy(labels), C).permute(2, 0, 1).double()
    back = lambda g: torch.einsum("Yh,cYX,Xw->chw", Mh, g, Mw) / (H * W)
    ref, A = back(p - oh), back(p + oh)
    K = band_grad_k(float(np.abs(lo).max()), C, band_extent(h, H), 2 * band_extent(w, W))
    return ref.numpy(), (K * U24 * A).numpy()


TEETH = [(6, 41, 128, 1024), (5, 36, 90, 713), (4, 25, 60, 473), (3, 65, 32, 1024), (3, 64, 16, 512), (4, 61, 64, 1024),
         (3, 20, 9, 83)]


@pytest.mark.parametrize("strip", [OHEM_STRIP, CE_STRIP])
@pytest.mark.parametrize("geom", TEETH, ids=["x".join(map(str, g)) for g in TEETH])
def test_bound_passes_emulation_and_rejects_mutants(geom, strip):
    h, H, w, W = geom
    rng = np.random.default_rng(h * W)
    C = 5
    lo = (rng.standard_normal((C, h, w)) * 2).astype(f32)
    labels = rng.integers(0, C, (H, W))
    ref, tol = _reference_and_bound(lo, labels)
    err = np.abs(_emulate_grad(lo, labels, strip) - ref)
    assert np.all(err <= tol), "honest emulation outside the bound by %g" % float((err / np.maximum(tol, 1e-300)).max())
    for mutant in ("drop_edge", "swap_clamped", "drop_last_row"):
        err = np.abs(_emulate_grad(lo, labels, strip, mutant) - ref)
        assert np.any(err > tol), "mutant %s passes the bound" % mutant
