"""Parity AT THE BASELINE SHAPE (BASELINE.json configs[1]: BiSeNet-R18, 16 x 1024 x 1024, 19 classes, OHEM): the whole
training step of the libtsb path against the oracle (oracle/torch_ref.py, bit-identical to the live reference modules)
run ON THE SAME GPU under stock torch.nn + cuDNN in strict fp32 (TF32 off) — SURVEY.md §8c "On the GPU box", north_star
"outputs match the reference PyTorch/cuDNN path".

The row-tile / resident-weight / persistent conv paths, the band OHEM kernels and the multi-wave streaming kernels only run at this
size, so this is where they are checked against the oracle (the small-shape tests exercise other tile choices).
Tolerances: loss 1e-2 (north_star, bf16); gradients of the business layers (heads, FFM, ARMs, refines, global context,
spatial path) norm_err <= 2e-2 per conv / classifier weight; BN running statistics 1e-2; the OHEM kept count of every
head equal to the oracle's."""
import pytest
import torch
import torch.nn.functional as F

from util import norm_err, make_labels

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d


def _oracle_kept_counts(lo, labels, min_kept):
    from oracle import torch_ref
    out = []
    for l, s in zip(lo, (16, 8, 8)):
        up = F.interpolate(l.detach(), scale_factor=s, mode="bilinear", align_corners=True)
        _, valid, thr = torch_ref.ohem_ce(up, labels, 255, 0.7, min_kept, return_aux=True)
        out.append((int(valid.sum()), float(thr)))
        del up
    return out


def test_bisenet_full_size_step_matches_oracle_cuda(cuda):
    import torchseg_b200
    from torchseg_b200 import ops
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight
    from oracle import torch_ref
    H = W = 1024
    free, _ = torch.cuda.mem_get_info()
    N = 16 if free > 120 * (1 << 30) else 8
    min_kept = N * H * W // 16                                   # train.py:48-49
    torch.manual_seed(12345)
    crit = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    crit.debug_states = []
    model = BiSeNet(19, True, crit, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    sd = {k: v.detach().clone().to(cuda) for k, v in model.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, 3, H, W, generator=g).to(cuda)
    y = make_labels(N, H, W, 19, 255, g).to(cuda)

    # ---- oracle on the GPU: stock torch.nn lowering, cuDNN, strict fp32
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark = True                        # train.py:35
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        stats = {}
        loss_ref, lo_ref = torch_ref.bisenet_r18_loss(x, y, sd, min_kept, stats=stats)
        loss_ref.backward()
        kept_ref = _oracle_kept_counts(lo_ref, y, min_kept)
        loss_ref_v = float(loss_ref)
        grads_ref = {k: v.grad.detach().cpu() for k, v in sd.items() if v.grad is not None}
        stats = {k: v.detach().cpu() for k, v in stats.items()}
        del loss_ref, lo_ref
        for v in sd.values():
            v.grad = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        # the SAME fp32 oracle with bf16 STORAGE emulated (values rounded to bf16 wherever the libtsb path stores bf16:
        # conv weights, raw conv outputs, activations — forward and backward). |fp32 − bf16-storage| is the spread that
        # the storage policy alone produces at this size; the libtsb step has to sit inside it.
        torch_ref.set_bf16_emulation(True)
        try:
            stats_emu = {}
            loss_emu, _ = torch_ref.bisenet_r18_loss(x, y, sd, min_kept, stats=stats_emu)
            loss_emu.backward()
        finally:
            torch_ref.set_bf16_emulation(False)
        loss_emu_v = float(loss_emu)
        grads_emu = {k: v.grad.detach().cpu() for k, v in sd.items() if v.grad is not None}
        stats_emu = {k: v.detach().cpu() for k, v in stats_emu.items()}
        del loss_emu
        for v in sd.values():
            v.grad = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old

    # ---- the libtsb step
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    loss = model(x, y)
    loss.backward()
    torch.cuda.synchronize()
    rel = abs(loss.item() - loss_ref_v) / abs(loss_ref_v)
    print("full-size N=%d: loss %.6f oracle %.6f rel %.2e (bf16-storage oracle %.6f)" % (N, loss.item(), loss_ref_v, rel, loss_emu_v))
    assert rel < 1e-2, (loss.item(), loss_ref_v)

    # OHEM: kept count per head (aux0, aux1, main — the order the network calls the criterion in). The whole-step counts
    # cannot be bit-equal: the two networks' logits differ by bf16-level noise, so the (few thousand) pixels whose p lies
    # within that noise of the 0.7 threshold flip. They must agree to 1e-3 here; the EXACT kept-set check at this size is
    # the teacher-forced test below (same logits into both).
    failures = []
    assert len(crit.debug_states) == 3
    for i, (st, (kept, thr)) in enumerate(zip(crit.debug_states, kept_ref)):
        d = ops.ohem_state_dict(st)
        n_kept = d["kept"]
        print("head %d: kept %d (oracle %d), threshold %.6f (oracle %.6f)" % (i, n_kept, kept, d["T"] if d["active"] else 0.7, thr))
        if abs(n_kept - kept) > 1e-3 * kept:
            failures.append(("kept", i, n_kept, kept))

    # gradients. An untrained batch-stat-BN network with random labels has gradients that are the small residue of
    # massive cancellation over 16.8 M pixels, and bf16 STORAGE alone moves them: `spread` = |oracle fp32 − the same oracle
    # with bf16 storage emulated|. The libtsb gradients must be as close to the fp32 oracle as that emulation is (x1.5 +
    # 2e-2), and closer to the emulation than the emulation is to fp32 wherever the spread is large.
    def _cos(a, b):
        a, b = a.reshape(-1), b.reshape(-1)
        return float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))

    business = ("spatial_path.", "global_context.", "arms.", "refines.", "heads.", "ffm.")
    rows, bad = [], []
    for n, p in model.named_parameters():
        a, b, c = p.grad.float().cpu(), grads_ref[n], grads_emu[n]
        e_ref, e_emu, spread = norm_err(a, b), norm_err(a, c), norm_err(c, b)
        rows.append((n, e_ref, e_emu, spread, _cos(a, b), _cos(c, b)))
        if p.dim() == 4 and e_ref > 1.5 * spread + 2e-2:
            bad.append((n, round(e_ref, 4), round(spread, 4)))
    print("%-46s %9s %9s %9s %8s %8s" % ("parameter", "err_fp32", "err_emu", "spread", "cos", "cos_emu"))
    for r in rows:
        if r[0].endswith("weight") and (r[0].startswith(business) or "conv" in r[0]):
            print("%-46s %9.4f %9.4f %9.4f %8.4f %8.4f" % r)
    worst = sorted(((r[1], r[0]) for r in rows), reverse=True)
    print("worst gradient norm_err vs fp32:", [(n, round(e, 4)) for e, n in worst[:8]])
    print("outside 1.5 x spread + 2e-2:", bad[:20])
    cos_bad = [(r[0], round(r[4], 4), round(r[5], 4)) for r in rows if r[4] < r[5] - 0.05]
    print("cosine below the emulation's by > 0.05:", cos_bad[:20])
    # the last classifier (one layer from the loss, nothing to amplify): tight
    e_cls = [r for r in rows if r[0] == "heads.2.conv_1x1.weight"][0][1]

    # BN running statistics (momentum 0.1, unbiased variance)
    msd = model.state_dict()
    stat_bad, stat_worst = [], 0.0
    for k, v in stats.items():
        den = v.abs().max().clamp_min(1e-6)
        e = float((msd[k].float().cpu() - v).abs().max() / den)
        spread = float((stats_emu[k] - v).abs().max() / den)
        stat_worst = max(stat_worst, e)
        if e >= 1e-2 + 1.5 * spread:
            stat_bad.append((k, round(e, 4), round(spread, 4)))
    print("running statistics: worst rel err %.4f; outside 1e-2 + 1.5 x spread: %s" % (stat_worst, stat_bad[:10]))
    assert not failures, failures
    assert not bad, "gradient farther from the fp32 oracle than 1.5 x the bf16-storage spread + 2e-2: %s" % bad[:10]
    assert not cos_bad, "gradient direction worse than the bf16-storage emulation's: %s" % cos_bad[:10]
    assert e_cls < 5e-2, e_cls
    assert not stat_bad, stat_bad[:10]


def test_ohem_full_size_kept_set_teacher_forced(cuda):
    """OHEM at the BASELINE size (16 x 19 x 1024 x 1024 after the x8 upsample) on IDENTICAL low-resolution logits: the
    fused-upsample kernels' kept set against torch's softmax / sort / threshold (the oracle restatement of
    loss_opr.py:68-98) evaluated on the same GPU. Two regimes: A (random logits: threshold 0.7, nearly all valid pixels
    kept) and B (confident logits: fewer than min_kept pixels below 0.7, so the threshold is the k-th smallest p).
    The pinned exp_det / ATen-order bilinear differ from torch's exp / FMA-contracted CUDA upsample in the last ulp, so a
    pixel whose p straddles the threshold within 1 ulp may flip: at most a handful out of 16.8 M (reported)."""
    from torchseg_b200 import ops
    from oracle import torch_ref
    N, C, h, w, s = 16, 19, 128, 128, 8
    H, W = h * s, w * s
    min_kept = N * H * W // 16
    g = torch.Generator().manual_seed(31)
    for regime in ("A", "B"):
        lo = torch.randn(N, C, h, w, generator=g)
        if regime == "A":
            labels = make_labels(N, H, W, C, 255, g).to(cuda)
        else:
            # confident logits on smooth label regions (64 x 64 low-res cells per class block): only the ~3 % of pixels
            # on block borders fall below 0.7 — fewer than min_kept = 1/16 of the pixels — so T = k-th smallest p > 0.7
            blocks = torch.randint(0, C, (N, h // 64, w // 64), generator=g)
            lab_lo = blocks.repeat_interleave(64, 1).repeat_interleave(64, 2)
            lo = lo + 9.0 * torch.nn.functional.one_hot(lab_lo, C).permute(0, 3, 1, 2).float()
            labels = lab_lo.repeat_interleave(s, 1).repeat_interleave(s, 2).contiguous()
            labels[:, : H // 10, :] = 255
            labels = labels.to(cuda)
        lo_d = ops.nhwc_zeros(N, C, h, w, dtype=torch.float32, device=cuda, cs=32)
        lo_d.copy_(lo.to(cuda))
        lo_d.requires_grad_(True)
        loss = ops.OhemUpCEFn.apply(lo_d, labels, H, W, C, 255, 0.7, min_kept, None)
        _, _, p, state, _ = loss.grad_fn.saved_tensors
        st = ops.ohem_state_dict(state)
        T = torch.tensor(st["T"], dtype=torch.float32, device=cuda)
        valid = labels.reshape(-1) != 255
        kept = valid & ((p <= T) if st["active"] else torch.ones_like(valid))
        up = F.interpolate(lo.to(cuda), scale_factor=s, mode="bilinear", align_corners=True)
        loss_ref, kept_ref, thr_ref = torch_ref.ohem_ce(up, labels, 255, 0.7, min_kept, return_aux=True)
        del up
        mism = int((kept != kept_ref.reshape(-1)).sum())
        print("regime %s: kept %d (oracle %d), mismatching pixels %d, T %.9g (oracle %.9g), loss %.6f (oracle %.6f)" % (
            regime, int(kept.sum()), int(kept_ref.sum()), mism, st["T"], thr_ref, loss.item(), float(loss_ref)))
        # torch's exp / FMA-contracted upsample vs the pinned recipe: <= a few ulp in p. In regime B ~1e6 pixels sit
        # within 5e-3 of T (density ~2e8 per unit p, i.e. ~12 pixels per ulp), so a few dozen may straddle it
        assert mism <= (8 if regime == "A" else 96), (regime, mism)
        assert abs(st["T"] - thr_ref) <= 1e-6 * max(1.0, abs(thr_ref)), (st["T"], thr_ref)
        assert abs(loss.item() - float(loss_ref)) < 1e-4 * abs(float(loss_ref))
        if regime == "B":
            assert st["active"] and st["T"] > 0.7 and abs(int(kept.sum()) - min_kept) <= 96
            # ... and BIT-EXACT against the C oracle (same pinned exp / bilinear recipe, oracle/tsb_oracle.c) at the full
            # 1024 x 1024 resolution on the first 4 images: p, T and the kept set must be identical
            import numpy as np
            from oracle import c_oracle
            n4 = 4
            mk4 = n4 * H * W // 16
            lo4 = ops.nhwc_zeros(n4, C, h, w, dtype=torch.float32, device=cuda, cs=32)
            lo4.copy_(lo[:n4].to(cuda))
            lab4 = labels[:n4].contiguous()
            loss4 = ops.OhemUpCEFn.apply(lo4.requires_grad_(True), lab4, H, W, C, 255, 0.7, mk4, None)
            _, _, p4, state4, _ = loss4.grad_fn.saved_tensors
            st4 = ops.ohem_state_dict(state4)
            lo_np = lo4.detach().permute(0, 2, 3, 1).cpu().numpy()           # [n, h, w, C] view of the NHWC buffer
            lo_np = np.ascontiguousarray(np.pad(lo_np, ((0, 0), (0, 0), (0, 0), (0, 32 - C))))
            up4 = c_oracle.bilinear_nhwc_to_nchw(lo_np, C, H, W)
            ref4 = c_oracle.ohem(up4, lab4.cpu().numpy(), 255, 0.7, mk4)
            p4 = p4.cpu().numpy()
            assert st4["active"] == ref4["active"]
            assert np.float32(st4["T"]).tobytes() == np.float32(ref4["T"]).tobytes(), (st4["T"], ref4["T"])
            assert np.array_equal(p4.view(np.uint32), ref4["p"].view(np.uint32)), "p_target bits differ from the C oracle"
            kept4 = (lab4.cpu().numpy().reshape(-1) != 255) & (p4 <= np.float32(st4["T"]))
            assert np.array_equal(kept4, ref4["kept"])
            assert abs(loss4.item() - ref4["loss"]) < 1e-5 * abs(ref4["loss"])
            print("regime B, 4 x 19 x 1024 x 1024 vs the C oracle: p bits, T bits and kept set (%d pixels) identical" % int(kept4.sum()))
