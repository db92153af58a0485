"""The eval-mode fold cache (ops._FoldCache) against the state it is built from, with the kernel calls mocked.

A training-mode forward updates the BN running statistics inside tsb_bn_finalize, through raw pointers that autograd's
version counters do not see. The fake finalize below writes them the same way (through `.data`, which shares the storage
but not the version counter), so these tests check that the finalize step (ops._bn_finalize, reached through
ops._bn_forward and the BiSeNet stem pair) makes the next eval-mode fold rebuild from the new statistics, for the plain,
stem and transposed folds."""
import pytest
import torch
import torch.nn as nn

KINDS = ["plain", "stem", "transposed"]


@pytest.fixture
def kernels(monkeypatch):
    """ops.call recorded by name; tsb_bn_finalize applies a fixed running-statistics update behind autograd's back"""
    from torchseg_b200 import ops
    calls = []

    def fake_call(name, *a):
        calls.append(name)
        if name == "tsb_bn_finalize" and a[12] is not None:
            a[12].data.add_(0.25)       # running_mean
            a[13].data.mul_(2.0)        # running_var

    monkeypatch.setattr(ops, "call", fake_call)
    monkeypatch.setattr(ops, "ptr", lambda t: t)
    monkeypatch.setattr(ops, "stream", lambda: 0)
    monkeypatch.setattr(ops, "det_ws", lambda: (0, 0))
    return calls


def _krsc(w):
    return w.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


def _layer(kind, seed):
    """(conv weight in KRSC storage, its BatchNorm with non-trivial statistics)"""
    g = torch.Generator().manual_seed(seed)
    K = 8
    shape = {"plain": (K, 16, 3, 3), "stem": (K, 3, 7, 7), "transposed": (16, K, 4, 4)}[kind]
    w = nn.Parameter(_krsc(torch.randn(shape, generator=g)))
    bn = nn.BatchNorm2d(K)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(K, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(K, generator=g))
        bn.running_mean.copy_(torch.randn(K, generator=g))
        bn.running_var.copy_(torch.rand(K, generator=g) + 0.5)
    return w, bn


def _folded_bias(bn):
    scale = bn.weight.float() / torch.sqrt(bn.running_var.float() + bn.eps)
    return bn.bias.float() - bn.running_mean.float() * scale


def _pack_calls(calls):
    return sum(n in ("tsb_pack_weight", "tsb_pack_stem_weight") for n in calls)


def _train_forward(kind, w, bn):
    """the running-statistics half of a training-mode forward of this layer, as the network runs it"""
    from torchseg_b200 import ops
    K = bn.num_features
    with torch.no_grad():
        if kind == "stem":   # BiSeNet's two 7x7/2 stems in one launch (ops.StemPairFn)
            w2, bn2 = _layer("stem", 99)
            xs = torch.zeros(2, 16, 4, 8)
            ops.StemPairFn.apply(xs, w, bn.weight, bn.bias, bn.running_mean, bn.running_var, w2, bn2.weight, bn2.bias,
                                 bn2.running_mean, bn2.running_var, 1e-5, 0.1, 1e-5, 0.1)
        else:                # ConvBNActFn (plain and transposed) and BNFn
            raw = ops.nhwc_empty(2, K, 4, 4, device="cpu")
            ops._bn_forward(raw, torch.zeros(2, K), 32.0, bn.weight, bn.bias, None, bn.running_mean, bn.running_var,
                            True, bn.eps, 0.1, True)


@pytest.mark.parametrize("kind", KINDS)
def test_fold_cache_rebuilds_after_training_forward(kernels, kind):
    from torchseg_b200 import ops
    w, bn = _layer(kind, 1)
    fc = ops._FoldCache()
    stem, tr = kind == "stem", kind == "transposed"
    wb, bias = fc.get(w, bn, stem, transposed=tr)
    assert torch.equal(bias, _folded_bias(bn)) and _pack_calls(kernels) == 1
    wb2, bias2 = fc.get(w, bn, stem, transposed=tr)
    assert wb2 is wb and bias2 is bias and _pack_calls(kernels) == 1, "a hit must return the cached tensors"
    rm_old = bn.running_mean.clone()
    _train_forward(kind, w, bn)
    assert not torch.equal(bn.running_mean, rm_old), "the fake finalize did not run"
    n = _pack_calls(kernels)
    wb3, bias3 = fc.get(w, bn, stem, transposed=tr)
    assert _pack_calls(kernels) == n + 1, "the fold was not rebuilt after the running statistics moved"
    assert wb3 is not wb and torch.equal(bias3, _folded_bias(bn))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("edit", ["conv_weight", "gamma", "beta", "running_mean", "running_var"])
def test_fold_cache_rebuilds_after_in_place_edit(kernels, kind, edit):
    from torchseg_b200 import ops
    w, bn = _layer(kind, 2)
    fc = ops._FoldCache()
    stem, tr = kind == "stem", kind == "transposed"
    wb, bias = fc.get(w, bn, stem, transposed=tr)
    t = {"conv_weight": w, "gamma": bn.weight, "beta": bn.bias, "running_mean": bn.running_mean,
         "running_var": bn.running_var}[edit]
    with torch.no_grad():
        t.mul_(1.5)
    wb2, bias2 = fc.get(w, bn, stem, transposed=tr)
    assert _pack_calls(kernels) == 2 and wb2 is not wb, edit
    assert torch.equal(bias2, _folded_bias(bn)), edit
    assert fc.get(w, bn, stem, transposed=tr)[1] is bias2 and _pack_calls(kernels) == 2
