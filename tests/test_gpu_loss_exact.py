"""Per-element checks of the loss kernels (ohem.cu, ce_up.cu, band.cuh, the focal kernel of pack_opt.cu) through the C ABI.

Buffers. Low-res logits are channels [OFF, OFF + C) of an NHWC buffer with channel stride cs > OFF + C; the other channels
hold NaN, so reading one poisons the result. Low-res gradient buffers start as a base pattern of small integers times a
power of two near the gradient's size (the up-sampled backward kernels add into the buffer), their pad channels hold a
NaN sentinel whose bits must come back unchanged, and the upstream gradient `gscale` is a device scalar other than 1.

References. OHEM p, T, `active` and the kept set come from the C oracle (bit for bit). Everything else is float64 torch on
the device fed the same fp32 inputs: up-sampling is the float64 matrix product with the kernels' fp32 lerp weights
(util.lerp_matrix, ATen's align_corners recipe), the gradient its adjoint. OHEM gradients use the oracle's kept set.

Tolerance: |got - ref| <= K * u * A + (final additions), u = 2^-24, A = the float64 sum of the absolute values of the
terms the kernel adds for that element. The kernels add the softmax part p and the one-hot part separately (the
one-hot part even through its own accumulator in ce_up), so A sums w_y * w_x * (p_c + [c = t]) * weight, not
|p_c - [c = t]|: that would understate the size of the terms where p_t is near 1. K follows from the kernel's roundings:
- blend: v = l0y * (l0x a + l1x b) + l1y * (...), separately rounded products and sums: |dv| <= 4 u M, M = max |logit|;
  the softmax of v + dv then has relative error <= 2 max|dv| = 8 u M;
- __expf(x) = ex2.approx(x * log2 e): the rounded product moves the result by a relative u |x|, ex2.approx adds <= 2^-22
  (4 u), the rounded argument x = v - m another u |x|; |x| <= 2 M, so <= u (4 M + 4) per exponential;
- the class sum: <= (C + 2) u; 1 / sum, the products with the pixel weight and gscale: <= 4 u;
  so OHEM's p has relative error <= u (12 M + C + 10);
- ce_up's backward forms p = exp(v - lse) with the forward's lse instead: the lse bound below (<= u (9 M + 2 C + 13),
  |lse| <= M + ln C), the blend's 4 u M, one exponential with |x| <= 2 M + 5 and 3 products: <= u (17 M + 2 C + 30);
- fmaf accumulation over the <= ny rows of a band and the <= nx strip columns of a low-res column pair: (ny + nx) u,
  and ce_up's one-hot tile, <= ny * nx shared-memory atomics per cell: ny * nx u; <= 4 global atomics per element: 4 u.
Hence K = 17 M + 2 C + ny + nx + ny nx + 34 (util.band_grad_k, the larger of the two), and the final additions onto the
base add 4 u (|base| + A). A per-pixel value (ce_up lse, OHEM nll) has error <= u (8 M + 2 C + 8 + |value|): the blend's
4 u M, one exponential's u (4 M + 4) times the sum's weights, the sum, logf and the last addition. A loss is a mean of
such values: the per-pixel bounds plus u (terms per thread + 8 levels of block_sum + 2) times the sum of |terms|.
The materialised OHEM gradient has no blend and no accumulation: K = 4 M + C + 12; bf16 adds one bf16 rounding.
The focal gradient has each term's error <= u (30 + 4 (gamma + 1) / (1 - s)): 1 - s loses the relative accuracy 4 u s
of s, and the terms raise it to the powers gamma - 1, gamma and 1; its loss sum adds one float atomic per block.

Integer outputs are exact: the ce_up count and 1/count, the OHEM num_valid / count_le / kept.
Labels must lie in [0, C) or equal the ignore label: the kernels index shared memory and class weights with them.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import U24, band_extent, band_grad_k, lerp_matrix
from test_cpu_band_geometry import MODEL_SHAPES, ce_up_fwd_ok, ohem_grad_up_path, ohem_ptarget_up_path

pytestmark = pytest.mark.gpu

F32, BF = torch.float32, torch.bfloat16
OFF = 5                        # channel offset of every low-res slice
SENT = 0x7FA5A5A5              # fp32 NaN bits no kernel computes
SENT_BF = 0x7FA5


def _ops():
    from torchseg_b200 import ops
    return ops


def _call(name, *args):
    ops = _ops()
    ops.call(name, *args, ops.stream())


def _launches():
    from torchseg_b200 import _lib
    return _lib.launch_count()


def _trip():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


# ------------------------------------------------------------------------------------------------ buffers
class LoBuf:
    """low-res NHWC [1, h, w, cs] with channels [OFF, OFF + C) live; inputs pad with NaN, gradients with SENT"""

    def __init__(self, h, w, C, vals=None, base=None):
        self.C, self.cs = C, OFF + C + 3
        if vals is not None:
            self.buf = torch.full((1, h, w, self.cs), float("nan"), dtype=F32, device="cuda")
            self.buf[..., OFF:OFF + C] = vals
        else:
            self.buf = torch.full((1, h, w, self.cs), SENT, dtype=torch.int32, device="cuda").view(F32)
            self.buf[..., OFF:OFF + C] = base

    @property
    def ptr(self):
        return self.buf.data_ptr() + 4 * OFF

    @property
    def v(self):
        return self.buf[..., OFF:OFF + self.C]

    def assert_pad(self, what):
        bits = self.buf.view(torch.int32)
        assert bool((bits[..., :OFF] == SENT).all()) and bool((bits[..., OFF + self.C:] == SENT).all()), \
            "%s: wrote outside the channel slice" % what


def _base_for(ref, g):
    """small integers times a power of two near max |ref|: the sum base + gradient keeps the gradient's precision"""
    e = math.frexp(max(float(ref.abs().max()), 1e-30))[1] - 3
    return torch.randint(-4, 5, tuple(ref.shape), generator=g, device="cuda").double() * 2.0 ** e


def _within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError("%s: %d of %d elements outside the bound, first at %s: got %s want %s tol %s" % (
            what, int(bad.sum()), got.numel(), idx, [float(got[tuple(i)]) for i in idx],
            [float(ref[tuple(i)]) for i in idx], [float(tol[tuple(i)]) for i in idx]))


def _grad_check(d, base, ref, A, K, what):
    """d: LoBuf after the kernel added into `base`; ref, A: [h, w, C] float64"""
    d.assert_pad(what)
    tol = K * U24 * A + 4 * U24 * (base.abs() + A)
    _within(d.v[0], base + ref, tol, what)


# ------------------------------------------------------------------------------------------------ float64 references
def _band_pass(lo, H, W, labels, per_pixel, rows=64):
    """Walk the up-sampled logits in row chunks. lo: [h, w, C] float64; per_pixel(up [C, y, W], lab [y, W], y0) returns
    a dict of [C, y, W] tensors to send back through the adjoint (summed into [h, w, C]) and of per-pixel tensors
    (concatenated)."""
    h, w, C = lo.shape
    Mh, Mw = lerp_matrix(h, H).cuda(), lerp_matrix(w, W).cuda()
    back, pix = {}, {}
    for y0 in range(0, H, rows):
        up = torch.einsum("yh,hwc,Xw->cyX", Mh[y0:y0 + rows], lo, Mw)
        out = per_pixel(up, labels[y0:y0 + rows], y0)
        for k, t in out.items():
            if t.dim() == 3:
                r = torch.einsum("yh,cyX,Xw->hwc", Mh[y0:y0 + rows], t, Mw)
                back[k] = back[k] + r if k in back else r
            else:
                pix.setdefault(k, []).append(t)
    return back, {k: torch.cat(v) for k, v in pix.items()}


def _softmax_parts(up, lab, valid, wt):
    C = up.shape[0]
    p = torch.softmax(up, dim=0)
    oh = F.one_hot(lab.clamp(0, C - 1), C).permute(2, 0, 1).double()
    m = valid.double() * wt
    return p, oh, m


def _pix_bound(M, C, val):
    return U24 * (8 * M + 2 * C + 8 + val.abs())


# ------------------------------------------------------------------------------------------------ ce_up
CE_CS = [1, 2, 5, 32, 33, 149, 150, 151, 152]
SMALL = [(12, 89, 40, 301), (1, 9, 1, 300), (7, 56, 3, 50), (5, 40, 33, 257), (3, 30, 9, 65), (6, 1, 30, 640),
         (4, 37, 2, 600), (9, 9, 20, 20), (2, 11, 64, 64)]
IGNS = [-1, 255, 0]


def _labels(H, W, C, ign, g):
    lab = torch.randint(0, C, (1, H, W), generator=g, device="cuda")
    drop = torch.rand(1, H, W, generator=g, device="cuda") < 0.07
    lab[drop] = ign
    lab[:, : max(0, H // 8 - 1)] = ign          # an ignored band at the top; the last row stays valid
    return lab


def _ce_up_case(C, h, H, w, W, ign, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo_v = (torch.randn(1, h, w, C, generator=g, device="cuda") * 2).float()
    labels = _labels(H, W, C, ign, g)
    lo = LoBuf(h, w, C, vals=lo_v)
    lse = torch.full((H * W,), float("nan"), device="cuda")
    state = torch.zeros(8, dtype=torch.int32, device="cuda")
    loss = torch.empty((), device="cuda")
    _call("tsb_ce_up_fwd", lo.ptr, lo.cs, h, w, labels.data_ptr(), 1, C, H, W, ign, lse.data_ptr(), state.data_ptr(),
          loss.data_ptr())
    gscale = torch.tensor(1.75, device="cuda")
    valid = labels[0] != ign
    count = int(valid.sum())
    M = float(lo_v.abs().max())
    wt = 1.75 / count if count else 0.0

    def per_pixel(up, lab, y0):
        v = lab != ign
        p, oh, m = _softmax_parts(up, lab, v, wt)
        lse_r = torch.logsumexp(up, dim=0)
        vt = up.gather(0, lab.clamp(0, C - 1)[None])[0]
        return dict(ref=(p - oh) * m, A=(p + oh) * m, lse=lse_r.reshape(-1), term=((lse_r - vt) * v).reshape(-1))

    back, pix = _band_pass(lo_v[0].double(), H, W, labels[0], per_pixel)
    # integer outputs
    st = state.cpu()
    assert int(st[2]) == count, "valid count"
    if count:
        assert st[4:5].view(torch.float32).item() == np.float32(1.0 / count), "1/count"
    # per-pixel lse, every pixel (ignored ones too)
    _within(lse, pix["lse"], _pix_bound(M, C, pix["lse"]), "ce_up lse C=%d %s" % (C, (h, H, w, W)))
    # loss
    ny = band_extent(h, H)
    if count:
        terms = pix["term"][valid.reshape(-1)]
        bound = (float(_pix_bound(M, C, pix["lse"])[valid.reshape(-1)].sum()) + 4 * U24 * M * count
                 + U24 * (ny + 10) * float(terms.abs().sum())) / count + 2 * U24 * float(terms.mean().abs())
        assert abs(loss.item() - float(terms.mean())) <= bound, ("ce_up loss", loss.item(), float(terms.mean()), bound)
    else:
        assert math.isnan(loss.item())
    # backward, adding into a base pattern
    ref, A = back["ref"], back["A"]
    base = _base_for(ref, g)
    d = LoBuf(h, w, C, base=base.float())
    _call("tsb_ce_up_bwd", lo.ptr, lo.cs, h, w, labels.data_ptr(), lse.data_ptr(), 1, C, H, W, ign, state.data_ptr(),
          gscale.data_ptr(), d.ptr)
    K = band_grad_k(M, C, ny, 2 * band_extent(w, W))
    _grad_check(d, base, ref, A, K, "ce_up grad C=%d %s" % (C, (h, H, w, W)))


def _ce_cases():
    out = []
    for i, C in enumerate(CE_CS):
        for j, (h, H, w, W) in enumerate(SMALL):
            if ce_up_fwd_ok(C, w, W):
                out.append((C, h, H, w, W, IGNS[(i + j) % 3]))
    return out


@pytest.mark.parametrize("case", _ce_cases(), ids=lambda c: "C%d_%dx%d_%dx%d_ign%d" % c)
def test_ce_up_small(cuda, case):
    C, h, H, w, W, ign = case
    _ce_up_case(C, h, H, w, W, ign, seed=C * 7 + W)


@pytest.mark.parametrize("shape", [s for s in MODEL_SHAPES if s[0] in (90, 60)] + [(16, 128, 16, 128)])
def test_ce_up_model_shapes(cuda, shape):
    h, H, w, W = shape
    _ce_up_case(150, h, H, w, W, -1, seed=h)


@pytest.mark.parametrize("C", CE_CS)
def test_ce_up_smallest_scale(cuda, C):
    """the smallest accepted W for w = 8 runs and is exact; one column less is refused with no launch"""
    w, h, H = 8, 3, 20
    W = next(W for W in range(1, 4000) if ce_up_fwd_ok(C, w, W))
    _ce_up_case(C, h, H, w, W, 255, seed=C)
    lo = LoBuf(h, w, C, vals=torch.zeros(1, h, w, C, device="cuda"))
    labels = torch.zeros(1, H, W - 1, dtype=torch.int64, device="cuda")
    lse = torch.empty(H * (W - 1), device="cuda")
    state = torch.zeros(8, dtype=torch.int32, device="cuda")
    n0 = _launches()
    with pytest.raises(RuntimeError, match="tsb_ce_up_fwd"):
        _call("tsb_ce_up_fwd", lo.ptr, lo.cs, h, w, labels.data_ptr(), 1, C, H, W - 1, 255, lse.data_ptr(),
              state.data_ptr(), None)
    assert _launches() == n0


# ------------------------------------------------------------------------------------------------ OHEM, up-sampled
OHEM_CS = [1, 2, 18, 19, 20, 21, 22, 31, 32]


def _ohem_forward_abi(pt, n, labels_ptr, ign, thresh, min_kept, cw):
    state = torch.empty(8192, dtype=torch.int32, device="cuda")
    p = torch.full((n,), float("nan"), device="cuda")
    nll = torch.full((n,), float("nan"), device="cuda")
    loss = torch.empty((), device="cuda")
    _call("tsb_ohem_begin", state.data_ptr())
    pt(p, nll, state)
    _call("tsb_ohem_select", p.data_ptr(), n, int(min_kept), float(thresh), state.data_ptr())
    _call("tsb_ohem_loss", p.data_ptr(), nll.data_ptr(), labels_ptr, n, ign, None if cw is None else cw.data_ptr(),
          state.data_ptr(), loss.data_ptr())
    return p, nll, state, loss


def _check_select(p, state, ref, labels_np, ign, thresh):
    ops = _ops()
    st = ops.ohem_state_dict(state)
    pn = p.cpu().numpy()
    assert np.array_equal(pn.view(np.uint32), ref["p"].view(np.uint32)), "p bits differ from the oracle"
    valid = labels_np.reshape(-1) != ign
    assert st["num_valid"] == int(valid.sum())
    assert st["count_le"] == int((ref["p"] <= np.float32(thresh)).sum())
    assert st["active"] == ref["active"]
    if ref["active"]:
        assert np.float32(st["T"]).view(np.uint32) == np.float32(ref["T"]).view(np.uint32)
    kept = valid & ((not st["active"]) | (pn <= np.float32(st["T"])))
    assert np.array_equal(kept, ref["kept"]), "kept set differs from the oracle"
    assert st["kept"] == int(ref["kept"].sum())
    return st


def _ohem_loss_check(loss, nll, ref, nll_r, labels, ign, cw, M, C, per_thread):
    """nll per pixel (0 where ignored) and the loss against float64 on the oracle's kept set"""
    kept = torch.from_numpy(ref["kept"]).cuda()
    lab = labels.reshape(-1)
    valid = lab != ign
    _within(nll, nll_r * valid, _pix_bound(M, C, nll_r) * valid, "OHEM nll")
    wts = (cw.double()[lab.clamp(0, C - 1)] if cw is not None else torch.ones_like(nll_r)) * kept
    if int(kept.sum()) == 0:
        assert math.isnan(loss.item())
        return 0.0
    den = float(wts.sum())
    ref_loss = float((wts * nll_r).sum()) / den
    bound = (float((wts * _pix_bound(M, C, nll_r)).sum()) + U24 * (per_thread + 12) * float((wts * nll_r.abs()).sum())) / den \
        + 2 * U24 * abs(ref_loss)
    assert abs(loss.item() - ref_loss) <= bound, ("OHEM loss", loss.item(), ref_loss, bound)
    return den


def _ohem_up_case(C, h, H, w, W, weighted, seed, min_kept_frac=16, twice=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo_v = (torch.randn(1, h, w, C, generator=g, device="cuda") * 2).float()
    labels = _labels(H, W, C, 255, g)
    lab_lo = labels[0, (torch.arange(h) * H // h).cuda()][:, (torch.arange(w) * W // w).cuda()].clamp(max=C - 1)
    lo_v[0] += 3 * F.one_hot(lab_lo, C).float()     # confident pixels: the select has to run for some cases
    cw = (torch.rand(C, generator=g, device="cuda") + 0.5) if weighted else None
    n = H * W
    min_kept = n // min_kept_frac
    lo = LoBuf(h, w, C, vals=lo_v)

    def pt(p, nll, state):
        _call("tsb_ohem_ptarget_up", lo.ptr, lo.cs, h, w, labels.data_ptr(), 1, C, H, W, 255, 0.7, p.data_ptr(),
              nll.data_ptr(), state.data_ptr())

    p, nll, state, loss = _ohem_forward_abi(pt, n, labels.data_ptr(), 255, 0.7, min_kept, cw)
    from oracle import c_oracle
    lab_np = labels.cpu().numpy()
    up = c_oracle.bilinear_nhwc_to_nchw(lo_v.cpu().numpy(), C, H, W)
    ref = c_oracle.ohem(up, lab_np, 255, 0.7, min_kept, class_weight=None if cw is None else cw.cpu().numpy())
    _check_select(p, state, ref, lab_np, 255, 0.7)
    M = float(lo_v.abs().max())
    kept = torch.from_numpy(ref["kept"]).cuda().reshape(H, W)
    lab = labels[0]

    def per_pixel(up64, lab_c, y0):
        k = kept[y0:y0 + up64.shape[1]]
        wt = (cw.double()[lab_c.clamp(0, C - 1)] if cw is not None else 1.0)
        p64, oh, m = _softmax_parts(up64, lab_c, k, wt)
        nll_r = torch.logsumexp(up64, dim=0) - up64.gather(0, lab_c.clamp(0, C - 1)[None])[0]
        return dict(ref=(p64 - oh) * m, A=(p64 + oh) * m, nll=nll_r.reshape(-1))

    back, pix = _band_pass(lo_v[0].double(), H, W, lab, per_pixel)
    den = _ohem_loss_check(loss, nll, ref, pix["nll"], labels, 255, cw, M, C, -(-n // _trip()) * 4)
    if den == 0:
        return
    gs = 0.625
    gscale = torch.tensor(gs, device="cuda")
    ref_g, A = back["ref"] * (gs / den), back["A"] * (gs / den)
    base = _base_for(ref_g, g)
    K = band_grad_k(M, C, band_extent(h, H), 2 * band_extent(w, W))
    outs = []
    for _ in range(2 if twice else 1):
        d = LoBuf(h, w, C, base=base.float())
        _call("tsb_ohem_grad_up", lo.ptr, lo.cs, h, w, labels.data_ptr(), p.data_ptr(), 1, C, H, W, 255,
              None if cw is None else cw.data_ptr(), state.data_ptr(), gscale.data_ptr(), d.ptr)
        _grad_check(d, base, ref_g, A, K,
                    "OHEM grad_up C=%d %s%s" % (C, (h, H, w, W), " weighted" if weighted else ""))
        outs.append(d.buf.clone())
    if twice:
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "exact-class gradient not deterministic"


def _ohem_cases():
    out = []
    for i, C in enumerate(OHEM_CS):
        for j, (h, H, w, W) in enumerate(SMALL):
            if ohem_ptarget_up_path(C, w, W) is not None:
                out.append((C, h, H, w, W, (i + j) % 2 == 1))
    return out


@pytest.mark.parametrize("case", _ohem_cases(), ids=lambda c: "C%d_%dx%d_%dx%d_%s" % (c[:5] + ("w" if c[5] else "u",)))
def test_ohem_up_small(cuda, case):
    C, h, H, w, W, weighted = case
    _ohem_up_case(C, h, H, w, W, weighted, seed=C * 13 + W,
                  twice=ohem_grad_up_path(C, w, W) == "x")


@pytest.mark.parametrize("C", [19, 21, 20])
def test_ohem_up_model_shape(cuda, C):
    """x8 at 1024 (one image): the exact-class kernels (19, 21) run twice and must agree bit for bit"""
    _ohem_up_case(C, 128, 1024, 128, 1024, C == 21, seed=C, min_kept_frac=2, twice=C != 20)


@pytest.mark.parametrize("shape", [s for s in MODEL_SHAPES if s[0] <= 64 and s[2] <= 128 and s[0] != 60])
def test_ohem_up_other_model_shapes(cuda, shape):
    h, H, w, W = shape
    _ohem_up_case(19, h, H, w, W, False, seed=W + h, twice=True)


def test_ohem_up_strips_sharing_columns(cuda):
    """w = 2, W = 600: strips 0 and 2 touch the same low-res columns, so C = 19 runs the generic gradient kernel"""
    assert ohem_grad_up_path(19, 2, 600) == "generic"
    _ohem_up_case(19, 3, 40, 2, 600, True, seed=600)


@pytest.mark.parametrize("C", OHEM_CS)
def test_ohem_up_smallest_scale(cuda, C):
    w, h, H = 8, 3, 20
    W = next(W for W in range(1, 4000) if ohem_ptarget_up_path(C, w, W) is not None)
    _ohem_up_case(C, h, H, w, W, False, seed=C + 1)
    if W > 1:
        lo = LoBuf(h, w, C, vals=torch.zeros(1, h, w, C, device="cuda"))
        labels = torch.zeros(1, H, W - 1, dtype=torch.int64, device="cuda")
        buf = torch.empty(H * (W - 1), device="cuda")
        state = torch.zeros(8192, dtype=torch.int32, device="cuda")
        n0 = _launches()
        with pytest.raises(RuntimeError, match="tsb_ohem_ptarget_up"):
            _call("tsb_ohem_ptarget_up", lo.ptr, lo.cs, h, w, labels.data_ptr(), 1, C, H, W - 1, 255, 0.7,
                  buf.data_ptr(), buf.data_ptr(), state.data_ptr())
        assert _launches() == n0


# ------------------------------------------------------------------------------------------------ OHEM, materialised
def _ohem_mat_case(C, H, W, dtype, layout, seed, labels=None, min_kept=None, thresh=0.7, lab_offset=False, cw=None,
                   logits=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if logits is None:
        logits = torch.randn(1, C, H, W, generator=g, device="cuda") * 2
        if labels is None:
            labels = _labels(H, W, C, 255, g)
        logits += 3 * F.one_hot(labels[0].clamp(0, C - 1), C).permute(2, 0, 1)[None] * (torch.rand(1, 1, H, W, generator=g, device="cuda") < 0.5)
    logits = logits.to(dtype).float()                        # the values the kernel reads, exactly
    n = H * W
    min_kept = n // 16 if min_kept is None else min_kept
    if lab_offset:                                           # labels 8 bytes off a 16-byte boundary: scalar loss path
        store = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        store[1:] = labels.reshape(-1)
        lab_ptr = store.data_ptr() + 8
    else:
        lab_ptr = labels.data_ptr()
    cs = OFF + C + 3
    if layout == "nchw":
        x = logits.to(dtype).contiguous()
        strides, xptr = x.stride(), x.data_ptr()
        dx = torch.full_like(x, float("nan"))
        dptr = dx.data_ptr()
        grad_of = lambda: dx[0].permute(1, 2, 0)
    else:                                                    # NHWC channel slice, as forward_lowres passes the classifier buffer
        buf = torch.full((1, H, W, cs), float("nan"), dtype=dtype, device="cuda")
        buf[..., OFF:OFF + C] = logits[0].permute(1, 2, 0).to(dtype)
        esz = buf.element_size()
        strides, xptr = (H * W * cs, 1, W * cs, cs), buf.data_ptr() + OFF * esz
        sent = SENT if dtype == F32 else SENT_BF
        bits = torch.int32 if dtype == F32 else torch.int16
        dbuf = torch.full((1, H, W, cs), sent, dtype=bits, device="cuda").view(dtype)
        dptr = dbuf.data_ptr() + OFF * esz
        grad_of = lambda: dbuf[0, :, :, OFF:OFF + C]
    dt = 0 if dtype == F32 else 1

    def pt(p, nll, state):
        _call("tsb_ohem_ptarget", xptr, dt, *strides, labels.data_ptr(), 1, C, H, W, 255, float(thresh), p.data_ptr(),
              nll.data_ptr(), state.data_ptr())

    p, nll, state, loss = _ohem_forward_abi(pt, n, lab_ptr, 255, thresh, min_kept, cw)
    from oracle import c_oracle
    lab_np = labels.cpu().numpy()
    ref = c_oracle.ohem(logits.cpu().numpy(), lab_np, 255, thresh, min_kept,
                        class_weight=None if cw is None else cw.cpu().numpy())
    st = _check_select(p, state, ref, lab_np, 255, thresh)
    up = logits[0].double()
    lab = labels[0]
    M = float(up.abs().max())
    nll_r = (torch.logsumexp(up, dim=0) - up.gather(0, lab.clamp(0, C - 1)[None])[0]).reshape(-1)
    den = _ohem_loss_check(loss, nll, ref, nll_r, labels, 255, cw, M, C, -(-n // _trip()) * 4)
    gs = 1.5
    gscale = torch.tensor(gs, device="cuda")
    _call("tsb_ohem_grad", xptr, dt, *strides, labels.data_ptr(), p.data_ptr(), 1, C, H, W, 255,
          None if cw is None else cw.data_ptr(), state.data_ptr(), gscale.data_ptr(), dptr)
    kept = torch.from_numpy(ref["kept"]).cuda().reshape(H, W)
    wt = (cw.double()[lab.clamp(0, C - 1)] if cw is not None else 1.0) * kept * (gs / den if den else 0.0)
    p64 = torch.softmax(up, dim=0)
    oh = F.one_hot(lab.clamp(0, C - 1), C).permute(2, 0, 1).double()
    ref_g = ((p64 - oh) * wt).permute(1, 2, 0)
    A = ((p64 + oh) * wt).permute(1, 2, 0)
    tol = (4 * M + C + 12) * U24 * A
    if dtype == BF:
        tol = tol + 2.0 ** -8 * (ref_g.abs() + tol)
    got = grad_of()
    _within(got.float(), ref_g, tol, "OHEM grad C=%d %s %s" % (C, layout, dtype))
    if layout == "nhwc":
        bits = dbuf.view(torch.int32 if dtype == F32 else torch.int16)
        sent = SENT if dtype == F32 else SENT_BF
        assert bool((bits[..., :OFF] == sent).all()) and bool((bits[..., OFF + C:] == sent).all()), "pad written"
    return st


@pytest.mark.parametrize("C", [19, 37, 150])
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_ohem_materialised(cuda, C, dtype, layout):
    cw = (torch.linspace(0.5, 2.0, C, device="cuda")) if C == 37 else None
    _ohem_mat_case(C, 37, 83, dtype, layout, seed=C + (dtype == BF), cw=cw)


# ------------------------------------------------------------------------------------------------ OHEM select edges
def _tie_logits(C, H, W, g, ndistinct=3):
    """every pixel takes one of `ndistinct` logit vectors, and labels from a short list: p has a handful of values"""
    pats = torch.randn(ndistinct, C, generator=g, device="cuda") * 2
    idx = torch.randint(0, ndistinct, (H, W), generator=g, device="cuda")
    logits = pats[idx].permute(2, 0, 1)[None].contiguous()
    labels = torch.randint(0, 2, (1, H, W), generator=g, device="cuda")
    return logits, labels


@pytest.mark.parametrize("which", ["k1", "nv-1", "nv", "nv+1"])
def test_ohem_select_ties_and_min_kept(cuda, which):
    g = torch.Generator(device="cuda").manual_seed(3)
    C, H, W = 19, 33, 61
    logits, labels = _tie_logits(C, H, W, g)
    labels[0, :4] = 255
    nv = int((labels != 255).sum())
    mk = {"k1": 1, "nv-1": nv - 1, "nv": nv, "nv+1": nv + 1}[which]
    st = _ohem_mat_case(C, H, W, F32, "nchw", 0, labels=labels, min_kept=mk, thresh=0.0, logits=logits)
    assert st["active"] == (mk <= nv)


@pytest.mark.parametrize("nb", ["below", "equal", "above"])
def test_ohem_thresh_at_the_kth_p(cuda, nb):
    from oracle import c_oracle
    g = torch.Generator(device="cuda").manual_seed(4)
    C, H, W = 19, 29, 47
    logits = torch.randn(1, C, H, W, generator=g, device="cuda") * 3
    labels = _labels(H, W, C, 255, g)
    k = H * W // 5
    ref = c_oracle.ohem(logits.cpu().numpy(), labels.cpu().numpy(), 255, 0.0, k)
    pk = np.sort(ref["p"])[k - 1]
    th = {"below": np.nextafter(pk, np.float32(-1)), "equal": pk, "above": np.nextafter(pk, np.float32(2))}[nb]
    st = _ohem_mat_case(C, H, W, F32, "nchw", 0, labels=labels, min_kept=k, thresh=float(th), logits=logits)
    assert np.float32(st["T"]) == max(np.float32(th), pk)


def test_ohem_every_label_ignored(cuda):
    g = torch.Generator(device="cuda").manual_seed(5)
    labels = torch.full((1, 21, 35), 255, dtype=torch.int64, device="cuda")
    st = _ohem_mat_case(19, 21, 35, F32, "nchw", 5, labels=labels)
    assert st["num_valid"] == 0 and not st["active"] and st["kept"] == 0


def test_ohem_multi_trip_odd_n_scalar_labels(cuda):
    """n > 3 trips of tsb_grid_for(n, 256, 8), n odd, labels off a 16-byte boundary (ohem_loss_kernel's scalar path)"""
    T = _trip()
    H, W = 3 * T // 901 + 7, 901
    _ohem_mat_case(19, H, W, F32, "nchw", 6, lab_offset=True)


def test_ohem_full_size_select_is_kthvalue(cuda):
    """16 x 19 x 1024 x 1024 up-sampled x8 with thresh 0: the three-level radix select runs on multi-trip grids, and T must
    equal torch.kthvalue of p (ignored pixels at 1) exactly"""
    N, C, h, w, s = 16, 19, 128, 128, 8
    H, W = h * s, w * s
    g = torch.Generator(device="cuda").manual_seed(1)
    lo = torch.randn(N, h, w, 32, device="cuda", generator=g) * 3
    labels = torch.randint(0, C, (N, H, W), device="cuda", generator=g)
    labels[:, :100] = 255
    n = N * H * W
    k = n // 16

    def pt(p, nll, state):
        _call("tsb_ohem_ptarget_up", lo.data_ptr(), 32, h, w, labels.data_ptr(), N, C, H, W, 255, 0.0, p.data_ptr(),
              nll.data_ptr(), state.data_ptr())

    p, nll, state, loss = _ohem_forward_abi(pt, n, labels.data_ptr(), 255, 0.0, k, None)
    st = _ops().ohem_state_dict(state)
    assert st["active"] and st["count_le"] < k
    kth = torch.kthvalue(p, k).values
    assert kth.view(torch.int32).item() == torch.tensor(st["T"], dtype=F32).view(torch.int32).item()
    valid = labels.reshape(-1) != 255
    assert st["num_valid"] == int(valid.sum())
    assert st["kept"] == int((valid & (p <= kth)).sum())


# ------------------------------------------------------------------------------------------------ focal
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("gamma,alpha", [(2.0, 0.25), (1.5, 0.6)])
def test_focal(cuda, dtype, gamma, alpha):
    n = 3 * _trip() + 12345
    g = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.randn(n, generator=g, device="cuda") * 2).clamp(-6, 6).to(dtype)
    t = torch.randint(0, 2, (n,), generator=g, device="cuda")
    t[torch.rand(n, generator=g, device="cuda") < 0.1] = 255
    loss = torch.zeros((), device="cuda")
    d = torch.full((n,), float("nan"), dtype=dtype, device="cuda")
    _call("tsb_sigmoid_focal_fwd_bwd", x.data_ptr(), 0 if dtype == F32 else 1, t.data_ptr(), n, 255, gamma, alpha,
          loss.data_ptr(), d.data_ptr())
    # float64 restatement of torch_ref.sigmoid_focal and of its derivative through s = sigmoid(x)
    xd = x.double()
    mask = (t != 255).double()
    y = t.double() * mask
    s = torch.sigmoid(xd)
    om = 1 - s
    lse = torch.log1p(torch.exp(-s))
    pos = om ** gamma * (s - s * y)
    neg = s ** gamma * lse
    l = -(alpha * pos + (1 - alpha) * neg) * mask
    dpos_a = gamma * om ** (gamma - 1) * (s - s * y)
    dpos_b = om ** gamma * (1 - y)
    dneg_a = gamma * s ** (gamma - 1) * lse
    dneg_b = s ** gamma * torch.exp(-s) / (1 + torch.exp(-s))
    chain = s * om / n * mask
    ref = -(alpha * (-dpos_a + dpos_b) + (1 - alpha) * (dneg_a - dneg_b)) * chain
    A = (alpha * (dpos_a + dpos_b) + (1 - alpha) * (dneg_a + dneg_b)) * chain
    tol = U24 * (30 + 4 * (gamma + 1) / om) * A
    if dtype == BF:
        tol = tol + 2.0 ** -8 * (ref.abs() + tol)
    _within(d.float(), ref, tol, "focal grad")
    ref_loss = float(l.sum()) / n
    blocks = torch.cuda.get_device_properties(0).multi_processor_count * 8
    lb = float((U24 * (30 + 4 * (gamma + 1) / om) * l.abs()).sum()) / n \
        + U24 * (-(-n // _trip()) + 8 + blocks) * float(l.abs().sum()) / n
    assert abs(loss.item() - ref_loss) <= lb, ("focal loss", loss.item(), ref_loss, lb)
