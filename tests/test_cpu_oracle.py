"""CPU tests: the oracle against the golden vectors generated from the LIVE reference (tools/make_golden.py,
tools/make_live_golden.py), and the two oracle restatements (C and
torch) against each other."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from golden_cases import ohem_case, bisenet_case, fcn_case, fcn_r101_case, pspnet_case, dfn_case, psanet_case, OHEM_REGIMES
from golden_cases import EVAL_KW, eval_image, eval_net, metric_inputs

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "reference_outputs.json")))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("regime", OHEM_REGIMES)
def test_c_oracle_ohem_vs_golden(regime):
    from oracle import c_oracle
    logits, labels, min_kept = ohem_case(regime)
    g = GOLD["ohem"][regime]
    out = c_oracle.ohem(logits.numpy(), labels.numpy(), 255, 0.7, min_kept, want_grad=True)
    if g["loss"] == "nan":
        assert np.isnan(out["loss"])
        return
    assert abs(out["loss"] - g["loss"]) < 1e-5 * abs(g["loss"])
    assert int(out["kept"].sum()) == g["kept_count"]
    assert _sha(out["kept"].astype(np.uint8)) == g["kept_sha256"], "kept index set differs from the reference"
    assert abs(float(np.abs(out["dlogits"]).sum()) - g["grad_abs_sum"]) < 1e-4 * g["grad_abs_sum"]


@pytest.mark.parametrize("regime", OHEM_REGIMES)
def test_torch_oracle_ohem_vs_golden_and_c(regime):
    from oracle import c_oracle, torch_ref
    logits, labels, min_kept = ohem_case(regime)
    g = GOLD["ohem"][regime]
    loss, valid, thr = torch_ref.ohem_ce(logits, labels, 255, 0.7, min_kept, return_aux=True)
    out = c_oracle.ohem(logits.numpy(), labels.numpy(), 255, 0.7, min_kept)
    if g["loss"] == "nan":
        assert torch.isnan(loss)
        return
    assert abs(float(loss) - g["loss"]) < 1e-6 * abs(g["loss"])
    assert np.array_equal(valid.numpy(), out["kept"])


def test_ohem_weighted_and_focal_vs_golden():
    from oracle import c_oracle, torch_ref
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    logits, labels, min_kept = ohem_case("B")
    w = np.array(ProbOhemCrossEntropy2d.CITYSCAPES_WEIGHT, np.float32)
    out = c_oracle.ohem(logits.numpy(), labels.numpy(), 255, 0.7, min_kept, class_weight=w)
    assert abs(out["loss"] - GOLD["ohem"]["B_weighted"]["loss"]) < 1e-5 * abs(GOLD["ohem"]["B_weighted"]["loss"])
    g = torch.Generator().manual_seed(10)
    pred = torch.randn(2, 1, 32, 40, generator=g)
    tgt = torch.randint(0, 2, (2, 32, 40), generator=g)
    tgt[:, :3] = 255
    assert abs(float(torch_ref.sigmoid_focal(pred, tgt, 255)) - GOLD["focal"]["loss"]) < 1e-6


def _ref_sd(build, seed):
    torch.manual_seed(seed)
    m = build()
    return m, {k: v.detach().clone() for k, v in m.state_dict().items()}


def test_torch_oracle_bisenet_vs_golden():
    """same seed → same initial weights (our module mirrors the reference's construction order) → same loss"""
    from oracle import torch_ref
    from torchseg_b200.networks import BiSeNet
    x, y, min_kept, seed = bisenet_case()
    m, sd = _ref_sd(lambda: BiSeNet(19, True, None, None, torch.nn.BatchNorm2d), seed)
    g = GOLD["bisenet_r18"]
    assert sum(p.numel() for p in m.parameters()) == g["n_params"] and len(sd) == g["n_state"]
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = torch_ref.bisenet_r18_loss(x, y, sd, min_kept)
    assert abs(float(loss) - g["loss"]) < 1e-5 * g["loss"]
    loss.backward()
    for n, ref in g["grad_norms"].items():
        assert abs(float(sd[n].grad.norm()) - ref) < 1e-4 * ref, n


def test_torch_oracle_fcn_r18_vs_golden():
    """BASELINE configs[0] (plumbing case): FCN-32s R18, 2 x 256 x 256, CPU"""
    from oracle import torch_ref
    from torchseg_b200.networks import FCN
    x, y, seed = fcn_case()
    torch.manual_seed(seed)
    m = FCN(19, backbone="R18")
    sd = {}
    for k, v in m.state_dict().items():   # reference key names: backbone.*, head.cbr.*, head.conv1x1.*
        sd[k] = v.detach().clone()
    loss = torch_ref.fcn_r18_loss(x, y, sd)
    assert abs(float(loss) - GOLD["fcn_r18"]["loss"]) < 1e-5 * GOLD["fcn_r18"]["loss"]


def test_torch_oracle_fcn_r101_vs_golden():
    """the shipped FCN-32s R101_v1c: our module reproduces the reference construction (seed → same weights, same keys)
    and the oracle restatement reproduces the live reference's loss / gradient norms"""
    from oracle import torch_ref
    from torchseg_b200.networks import FCN
    x, y, seed = fcn_r101_case()
    torch.manual_seed(seed)
    m = FCN(21, torch.nn.CrossEntropyLoss(ignore_index=255), backbone="R101")
    g = GOLD["fcn_r101"]
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    assert sum(p.numel() for p in m.parameters()) == g["n_params"] and len(sd) == g["n_state"]
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = torch_ref.fcn_r101_loss(x, y, sd)
    assert abs(float(loss) - g["loss"]) < 1e-5 * g["loss"]
    loss.backward()
    for n, ref in g["grad_norms"].items():
        assert abs(float(sd[n].grad.norm()) - ref) < 1e-4 * ref, n


def test_torch_oracle_pspnet_vs_golden():
    """PSPNet-R101_v1c dilated-8: our module reproduces the reference construction (same seed → same weights, same
    state_dict keys) and the oracle restatement reproduces the live reference's loss / gradient norms"""
    from oracle import torch_ref
    from torchseg_b200.networks import PSPNet
    x, y, seed = pspnet_case()
    torch.manual_seed(seed)
    m = PSPNet(150, torch.nn.CrossEntropyLoss(ignore_index=-1))
    g = GOLD["pspnet_r101"]
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    assert sum(p.numel() for p in m.parameters()) == g["n_params"] and len(sd) == g["n_state"]
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = torch_ref.pspnet_loss(x, y, sd)
    assert abs(float(loss) - g["loss"]) < 1e-5 * g["loss"]
    loss.backward()
    for n, ref in g["grad_norms"].items():
        assert abs(float(sd[n].grad.norm()) - ref) < 1e-4 * ref, n


def test_torch_oracle_dfn_vs_golden():
    """DFN-R101_v1c: module construction (seed → same weights / keys / 90.22 M params) and the oracle restatement of
    RefineResidual / ChannelAttention / DFNHead / DFN.forward against the live reference's loss and gradient norms"""
    from oracle import torch_ref
    from torchseg_b200.networks import DFN
    from torchseg_b200.seg_opr.loss_opr import SigmoidFocalLoss
    x, y, e, seed = dfn_case()
    torch.manual_seed(seed)
    m = DFN(19, torch.nn.CrossEntropyLoss(ignore_index=255), SigmoidFocalLoss(255), 0.1)
    g = GOLD["dfn_r101"]
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    assert sum(p.numel() for p in m.parameters()) == g["n_params"] and len(sd) == g["n_state"]
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = torch_ref.dfn_loss(x, y, e, sd)
    assert abs(float(loss) - g["loss"]) < 1e-5 * g["loss"]
    loss.backward()
    for n, ref in g["grad_norms"].items():
        assert abs(float(sd[n].grad.norm()) - ref) < 1e-4 * ref, n


def test_torch_oracle_psanet_vs_golden():
    """PSANet-R101_v1c (SURVEY C5): construction parity (79.58 M params, 684 state entries) and the oracle restatement
    of PointwiseSpatialAttention (softmax over the 3600 attention channels + bmm) against the live reference"""
    from oracle import torch_ref
    from torchseg_b200.networks import PSANet
    x, y, seed = psanet_case()
    torch.manual_seed(seed)
    m = PSANet(150, torch.nn.CrossEntropyLoss(ignore_index=-1))
    g = GOLD["psanet_r101"]
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    assert sum(p.numel() for p in m.parameters()) == g["n_params"] and len(sd) == g["n_state"]
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = torch_ref.psanet_loss(x, y, sd)
    assert abs(float(loss) - g["loss"]) < 1e-5 * g["loss"]
    loss.backward()
    for n, ref in g["grad_norms"].items():
        assert abs(float(sd[n].grad.norm()) - ref) < 1e-4 * ref, n


def test_exp_det_properties():
    from oracle import c_oracle
    assert c_oracle.exp_det(0.0) == 1.0
    assert c_oracle.exp_det(-200.0) == 0.0
    xs = np.linspace(-80, 0, 2001).astype(np.float32)
    e = np.array([c_oracle.exp_det(float(v)) for v in xs])
    r = np.exp(xs.astype(np.float64))
    assert np.max(np.abs(e - r) / r) < 4e-7
    assert np.all(np.diff(e) >= 0)  # monotone


def test_bilinear_oracle_matches_aten():
    from oracle import c_oracle
    g = torch.Generator().manual_seed(4)
    lo = torch.randn(2, 6, 9, 32, generator=g)
    ref = torch.nn.functional.interpolate(lo[..., :19].permute(0, 3, 1, 2), scale_factor=8, mode="bilinear", align_corners=True)
    out = c_oracle.bilinear_nhwc_to_nchw(lo.numpy(), 19, 48, 72)
    assert np.max(np.abs(out - ref.numpy())) < 1e-5


@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "weighted"])
def test_ohem_extra_masked_class_changes_nothing(weighted):
    """An extra class whose low-res logit is -1e4 and that no label names leaves the fused-upsample OHEM bit-identical:
    its exp flushes to exactly 0 and adding +0 leaves every class-order sum unchanged, so p, T, the kept set, the loss
    and the gradient of the real classes are the same, and the extra class's gradient is 0. test_gpu_kernels.py relies
    on this to run the same 19-class input through the generic band kernels (as C = 20)."""
    from oracle import c_oracle
    N, C, h, w, s = 2, 19, 12, 16, 8
    H, W = h * s, w * s
    g = torch.Generator().manual_seed(31)
    lo = torch.randn(N, h, w, 32, generator=g) * 3
    lo[..., C] = -1e4
    labels = torch.randint(0, C, (N, H, W), generator=g)
    labels[:, :10] = 255
    cw = (torch.rand(C + 1, generator=g) + 0.5).numpy() if weighted else None
    min_kept = N * H * W // 16
    res = []
    for c in (C, C + 1):
        up = c_oracle.bilinear_nhwc_to_nchw(lo.numpy(), c, H, W)
        res.append(c_oracle.ohem(up, labels.numpy(), 255, 0.7, min_kept, class_weight=None if cw is None else cw[:c],
                                 want_grad=True))
    a, b = res
    assert np.array_equal(a["p"].view(np.uint32), b["p"].view(np.uint32))
    assert np.array_equal(a["kept"], b["kept"])
    assert a["T"] == b["T"] and a["active"] == b["active"] and a["loss"] == b["loss"]
    assert np.array_equal(a["dlogits"].view(np.uint32), np.ascontiguousarray(b["dlogits"][:, :C]).view(np.uint32))
    assert np.all(b["dlogits"][:, C] == 0)


# ---------------------------------------------------------------------------------------------------------------
# the reference modules' own outputs, stored by tools/make_live_golden.py (tests/golden/live_reference.npz)
# ---------------------------------------------------------------------------------------------------------------
LIVE = np.load(os.path.join(HERE, "golden", "live_reference.npz"))


def test_oracle_vs_live_reference_ohem():
    from oracle import c_oracle
    for regime in ["A", "B", "C", "D"]:
        for seed in (1, 2, 3):
            k = "ohem_%s%d_" % (regime, seed)
            logits, labels, min_kept = ohem_case(regime, seed=seed, H=32, W=40)
            out = c_oracle.ohem(logits.numpy(), labels.numpy(), 255, 0.7, min_kept, want_grad=True)
            assert np.array_equal(out["kept"], LIVE[k + "kept"]), (regime, seed)
            loss = float(LIVE[k + "loss"])
            assert abs(out["loss"] - loss) < 1e-5 * abs(loss)
            assert np.max(np.abs(out["dlogits"].reshape(-1)[LIVE[k + "grad_idx"]] - LIVE[k + "grad"])) < 1e-6


def test_oracle_vs_live_reference_bisenet_exact():
    from oracle import torch_ref
    from torchseg_b200.networks import BiSeNet
    x, y, min_kept, seed = bisenet_case(N=2, HW=64, seed=5)
    torch.manual_seed(seed)
    m = BiSeNet(19, True, None, None, torch.nn.BatchNorm2d)   # same seed → the reference's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = torch_ref.bisenet_r18_loss(x, y, sd, min_kept)
    loss.backward()
    assert float(loss) == float(LIVE["bisenet_loss"])
    for n, (norm, idx, vals) in json.loads(str(LIVE["bisenet_grads"])).items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_module_key_names_match_reference():
    """checkpoint compatibility: our BiSeNet exposes exactly the reference's state_dict keys and shapes (App. D)"""
    from torchseg_b200.networks import BiSeNet
    ref = json.loads(str(LIVE["bisenet_keys"]))
    ours = BiSeNet(19, True, None, None, torch.nn.BatchNorm2d).state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_metric_functions_vs_live_reference():
    """seg_opr.metric (confusion matrix / IoU / ADE intersection-union) against the reference's metric.py on seeded
    predictions, incl. ignore labels (255 → outside [0, n_cl), -1 for ADE) and classes that never occur"""
    from torchseg_b200.seg_opr import metric as mine
    n_cl, pred, gt, pr, lab = metric_inputs()
    h2, l2, c2 = LIVE["metric_hist"], int(LIVE["metric_labeled"]), int(LIVE["metric_correct"])
    h1, l1, c1 = mine.hist_info(n_cl, pred, gt)
    assert np.array_equal(h1, h2) and l1 == l2 and c1 == c2
    for i, a in enumerate(mine.compute_score(h1, c1, l1)):
        assert np.allclose(a, LIVE["metric_score_%d" % i], equal_nan=True)
    ht, lt, ct = mine.hist_info_torch(n_cl, torch.from_numpy(pred), torch.from_numpy(gt))
    assert np.array_equal(ht.numpy(), h2) and int(lt) == l2 and int(ct) == c2
    # ADE protocol
    i1, u1 = mine.intersectionAndUnion(pr, lab, 150)
    assert np.array_equal(i1, LIVE["metric_inter"]) and np.array_equal(u1, LIVE["metric_union"])
    for i, a in enumerate(mine.meanIoU(np.stack([i1, i1], 1), np.stack([u1, u1], 1))):
        assert np.allclose(a, LIVE["metric_miou_%d" % i], equal_nan=True)
    assert np.array_equal(np.asarray(mine.pixelAccuracy(pr, lab), dtype=np.float64), LIVE["metric_pixacc"])
    assert mine.mean_pixel_accuracy([3, 4], [5, 6]) == float(LIVE["metric_mpa"])
    assert mine.accuracy(pr, lab)[0] == float(LIVE["metric_acc"])


def test_evaluator_sliding_and_whole_eval_vs_live_reference(monkeypatch):
    """engine.evaluator (batched sliding-window evaluation) against the reference Evaluator run on the CPU with a small
    deterministic network: same window grid, same summed (not averaged) overlap handling, same flip / multi-scale
    accumulation, same cv2 resizes → identical arg-max maps and matching scores"""
    from torchseg_b200.engine.evaluator import Evaluator
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self, raising=False)
    mine = Evaluator(crop_batch=3, **EVAL_KW)
    mine.val_func = eval_net()
    img = eval_image()
    # sliding evaluation: crop 96 on a 150x210 image → 2x3 .. 3x5 windows per scale, incl. the single-window scale path
    p_mine = mine.sliding_eval(img, 96, 2 / 3.0, None)
    assert p_mine.shape == (150, 210)
    assert (LIVE["eval_sliding"] == p_mine).mean() > 0.999
    s_mine = mine.scale_process(img, (150, 210), 96, 2 / 3.0, None)
    assert np.abs(s_mine.reshape(-1)[LIVE["eval_scale_idx"]] - LIVE["eval_scale"]).max() < 1e-4 * float(LIVE["eval_scale_absmax"])
    assert mine.window_grid(150, 210, 96, 2 / 3.0) == [(0, 0), (0, 64), (0, 114), (54, 0), (54, 64), (54, 114)]
    # small image → single padded window
    assert np.array_equal(LIVE["eval_small"], mine.sliding_eval(img[:80, :70], 96, 2 / 3.0, None))
    # whole-image evaluation with padding to a fixed input size and resize to an output size
    assert (LIVE["eval_whole"] == mine.whole_eval(img, (75, 105), (160, 224), None)).mean() > 0.999
    # grey-scale input path
    assert (LIVE["eval_grey"] == mine.whole_eval(img[:, :, :1], None, None, None)).mean() > 0.999


def test_oracle_dfn_blocks_vs_live_reference_modules():
    """RefineResidual / BNRefine / ChannelAttention restatements against the reference modules' outputs (bit-exact, fp32)"""
    from oracle import torch_ref as tr

    def sd_of(key):
        return {"m." + k: torch.tensor(v, dtype=torch.float32 if isinstance(v, list) else None)
                for k, v in json.loads(str(LIVE[key])).items()}
    x, x2 = torch.from_numpy(LIVE["dfn_x"]), torch.from_numpy(LIVE["dfn_x2"])
    for relu in (True, False):
        out = tr.bn_refine(x, sd_of("dfn_bnrefine_%d_sd" % relu), "m", relu, 1e-5, 0.1, True)
        assert torch.equal(out, torch.from_numpy(LIVE["dfn_bnrefine_%d_out" % relu]))
        out = tr.refine_residual(x, sd_of("dfn_refres_%d_sd" % relu), "m", relu, 1e-5, 0.1, True)
        assert torch.equal(out, torch.from_numpy(LIVE["dfn_refres_%d_out" % relu]))
    out = tr.channel_attention(x, x2, sd_of("dfn_ca_sd"), "m")
    assert torch.allclose(out, torch.from_numpy(LIVE["dfn_ca_out"]), atol=1e-6)
