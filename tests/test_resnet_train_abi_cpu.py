"""CPU tests of ResNet-trunk training (frcnn_b200/resnet_train.py):
  * the four new entries (frcnn_maxpool3x3s2_backward, frcnn_grad_prepare_stride2, frcnn_fold_batchnorm,
    frcnn_wgrad_reduce_scaled) are exported with their declared signatures and reject bad arguments with FRCNN_ERR_ARG
    before anything touches the device (the pointers are fake and never dereferenced);
  * ResNetRpnTrainer rejects bad options and parameters before it allocates anything;
  * the restatements of the two re-layouts (tests/resnet_train_ref.py) agree with torch autograd on tie-free inputs;
  * the oracle's frozen-BN step: the gradients of the unfolded BN graph equal s * the folded convolution's gradients."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import frcnn_oracle as orc
import resnet_train_oracle as rto
import resnet_train_ref as rtr
from resnet_ref import maxpool_cover_all, split_rne
from test_train_targets_abi_cpu import P, _fail, _params

ERR_ARG = -1
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
NAMES = ("frcnn_maxpool3x3s2_backward", "frcnn_grad_prepare_stride2", "frcnn_fold_batchnorm", "frcnn_wgrad_reduce_scaled")


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "double": ctypes.c_double, "float": ctypes.c_float}
    for name in NAMES:
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
        assert res is ctypes.c_int, name


def _pool(lib, g=P, y=P, p=P, H=9, W=7, C=64, o=P, t=None):
    return lib.frcnn_maxpool3x3s2_backward(g, None, y, None, p, None, H, W, C, o, None, t, None, None)


@pytest.mark.parametrize("kw,words", [
    (dict(g=None), ["maxpool3x3s2_backward"]),
    (dict(y=None), ["maxpool3x3s2_backward"]),
    (dict(p=None), ["maxpool3x3s2_backward"]),
    (dict(H=1), ["maxpool3x3s2_backward", "H=1"]),
    (dict(W=0), ["maxpool3x3s2_backward"]),
    (dict(C=12), ["maxpool3x3s2_backward", "C=12"]),
    (dict(o=None), ["no output"]),
])
def test_maxpool3x3s2_backward_errors(lib, kw, words):
    _fail(_pool(lib, **kw), ERR_ARG, words)


def _s2(lib, g=P, H=9, W=7, C=64, o=P, t=None, planes=1):
    return lib.frcnn_grad_prepare_stride2(g, None, P, None, H, W, C, o, None, t, None, planes, None)


@pytest.mark.parametrize("kw,words", [
    (dict(g=None), ["grad_prepare_stride2"]),
    (dict(H=0), ["grad_prepare_stride2", "H=0"]),
    (dict(C=20), ["grad_prepare_stride2", "C=20"]),
    (dict(planes=2), ["planes"]),
    (dict(o=None), ["no output"]),
])
def test_grad_prepare_stride2_errors(lib, kw, words):
    _fail(_s2(lib, **kw), ERR_ARG, words)


@pytest.mark.parametrize("kw,words", [
    (dict(w=None), ["fold_batchnorm", "NULL"]),
    (dict(s=None), ["fold_batchnorm", "NULL"]),
    (dict(wf=None), ["fold_batchnorm", "NULL"]),
    (dict(Cout=0), ["fold_batchnorm", "Cout=0"]),
    (dict(per_out=0), ["fold_batchnorm", "per_out=0"]),
    (dict(beta=None), ["beta and mean"]),
])
def test_fold_batchnorm_errors(lib, kw, words):
    a = dict(w=P, s=P, Cout=64, per_out=147, b=P, beta=P, mean=P, wf=P, bf=P)
    a.update(kw)
    _fail(lib.frcnn_fold_batchnorm(a["w"], a["s"], a["Cout"], a["per_out"], a["b"], a["beta"], a["mean"], a["wf"], a["bf"], None),
          ERR_ARG, words)


@pytest.mark.parametrize("kw,words", [
    (dict(parts=None), ["wgrad_reduce_scaled", "NULL"]),
    (dict(s=None), ["wgrad_reduce_scaled", "NULL"]),
    (dict(dw=None), ["wgrad_reduce_scaled", "NULL"]),
    (dict(groups=0), ["groups=0"]),
    (dict(splits=0), ["splits=0"]),
    (dict(M_parts=63), ["M_parts=63"]),
    (dict(ld=31), ["ld=31"]),
])
def test_wgrad_reduce_scaled_errors(lib, kw, words):
    a = dict(parts=P, groups=9, splits=2, M_parts=64, M=64, ld=32, N=32, s=P, dw=P)
    a.update(kw)
    _fail(lib.frcnn_wgrad_reduce_scaled(a["parts"], a["groups"], a["splits"], a["M_parts"], a["M"], a["ld"], a["N"], a["s"], a["dw"],
                                        None), ERR_ARG, words)


@pytest.fixture(scope="module")
def r50():
    return orc.make_resnet_params(n_layers=50, seed=11)


@pytest.mark.parametrize("kw,words", [
    (dict(n_layers=34), ["n_layers"]),
    (dict(subsample="random"), ["subsample"]),
    (dict(feat_stride=16), ["feat_stride"]),
    (dict(H=4), ["5 x 5"]),
    (dict(precision="fp8"), ["precision"]),
])
def test_trainer_rejects_bad_options(r50, kw, words):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    a = dict(H=64, W=96, n_layers=50)
    a.update(kw)
    H, W = a.pop("H"), a.pop("W")
    with pytest.raises(FrcnnError) as e:
        ResNetRpnTrainer(r50, H, W, ANCHORS, **a)
    assert all(w in str(e.value) for w in words), str(e.value)


@pytest.mark.parametrize("drop,shape", [("trunk/res3/a/bn4/avg_var", None), ("trunk/res4/b2/conv2/W", (256, 256, 1, 1)),
                                        ("RPN/rpn_conv_3x3/W", (512, 1024, 3, 3))])
def test_trainer_rejects_bad_parameters(r50, drop, shape):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    p = dict(r50)
    if shape is None:
        del p[drop]
    else:
        p[drop] = np.zeros(shape, np.float32)
    with pytest.raises(FrcnnError, match=drop):
        ResNetRpnTrainer(p, 64, 96, ANCHORS, n_layers=50)


def _tie_free(shape, seed, positive_share=0.7):
    """float32 values, distinct in every window, about positive_share of them > 0, exactly representable in bf16 pairs."""
    g = torch.Generator().manual_seed(seed)
    n = int(np.prod(shape))
    v = (torch.randperm(4 * n, generator=g)[:n].float() + 1.0) / 64.0
    v = torch.where(torch.rand(n, generator=g) < positive_share, v, -v)
    return v.view(shape)


@pytest.mark.parametrize("H,W", [(3, 3), (4, 5), (7, 6), (9, 9), (12, 17)])
def test_pool_backward_restatement_matches_autograd(H, W):
    C = 8
    y = torch.relu(_tie_free((H, W, C), H * 31 + W))             # post-ReLU: zeros tie, but a 0 element is masked anyway
    y_hi, y_lo = split_rne(y)
    p = maxpool_cover_all(rtr.pair_f32(y_hi, y_lo)).float()
    p_hi, p_lo = split_rne(p)
    gv = _tie_free(p.shape, 7, positive_share=0.5)
    g_hi, g_lo = split_rne(gv)
    hi, lo = rtr.maxpool3x3s2_backward(g_hi, g_lo, y_hi, y_lo, p_hi, p_lo)
    got = rtr.pair_f32(hi, lo).double()
    x = rtr.pair_f32(y_hi, y_lo).double().permute(2, 0, 1)[None].requires_grad_(True)
    out = F.max_pool2d(x, 3, 2, ceil_mode=True)
    assert tuple(out.shape[2:]) == tuple(p.shape[:2])
    out.backward(rtr.pair_f32(g_hi, g_lo).double().permute(2, 0, 1)[None])
    want = (x.grad[0] * (x[0] > 0)).permute(1, 2, 0)
    torch.testing.assert_close(got, want, rtol=1e-6, atol=0)
    assert torch.count_nonzero(got) > 0


@pytest.mark.parametrize("H,W", [(1, 1), (2, 3), (5, 4), (8, 8), (11, 6)])
@pytest.mark.parametrize("masked", [False, True])
def test_stride2_restatement_matches_autograd(H, W, masked):
    C = 16
    g = _tie_free(((H + 1) // 2, (W + 1) // 2, C), H + W, positive_share=0.5)
    g_hi, g_lo = split_rne(g)
    y = torch.relu(_tie_free((H, W, C), 3 * H + W))
    y_hi, _ = split_rne(y)
    hi, lo = rtr.grad_prepare_stride2(g_hi, g_lo, H, W, y_hi if masked else None)
    x = torch.zeros((H, W, C), dtype=torch.float64, requires_grad=True)
    x[0::2, 0::2].backward(rtr.pair_f32(g_hi, g_lo).double())
    want = x.grad * (y_hi.double() > 0) if masked else x.grad
    assert torch.equal(rtr.pair_f32(hi, lo).double(), want)


def test_transposed_layout():
    a = torch.arange(1, 3 * 5 * 8 + 1, dtype=torch.float32).view(3, 5, 8).to(torch.bfloat16)
    Kp, Wp = rtr.padded_pixels(3, 5)
    assert (Kp, Wp) == (128, 16)
    t = rtr.transposed(a, 3)
    assert t.shape == (3, 8, Kp)
    assert t[1, 2, 2 * Wp + 8 + 4] == a[1, 4, 2] and t[0, 2, 2 * Wp + 8 + 4] == a[1, 3, 2] and t[2, 2, 2 * Wp + 8 + 3] == a[1, 4, 2]
    assert t[2, 2, 2 * Wp + 8 + 4] == 0 and t[0, 2, 2 * Wp + 8] == 0
    assert t[0, 2, 2 * Wp + 8 + 5] == a[1, 4, 2] and t[0, 2, 2 * Wp + 8 + 6] == 0      # the 8-pixel group past the map
    assert torch.count_nonzero(t[1]) == a.numel() and torch.count_nonzero(t[0]) == a.numel()


def test_oracle_frozen_bn_gradients_are_scaled_folded_gradients(r50):
    """resnet_rpn_train_step at ResNet-50 on a 128 x 160 image: dL/dW of the unfolded graph (conv, then the BN formula with
    constant statistics) equals s * dL/dWf of the folded one in float64, for every trunk convolution and conv1's bias."""
    H, W = 128, 160
    x = orc.make_image(H, W, seed=5)
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(2, 4, 8))
    fh, fw = 4, 5
    gt = np.array([[[10, 8, 60, 50, 3], [40, 30, 150, 120, 7]]], np.float32)
    r = orc.anchor_target_layer(fh, fw, gt, np.array([[H, W]], np.int32), anchors=anchors, feat_stride=32, choice=lambda a, n: a[:0])
    args = (r50, x, r["labels_before_subsample"], r["targets"], r["inds_inside"])
    a = rto.resnet_rpn_train_step(*args, n_layers=50)
    b = rto.resnet_rpn_train_step(*args, n_layers=50, folded=True)
    assert np.allclose(a["losses"], b["losses"], rtol=1e-12, atol=0)
    assert set(a["grads"]) == set(b["grads"])
    assert "trunk/conv1/b" in a["grads"] and not any("/bn" in k for k in a["grads"])
    worst = 0.0
    for k in a["grads"]:
        ga, gb = a["grads"][k], b["grads"][k]
        assert np.abs(ga).max() > 0, k
        worst = max(worst, float(np.abs(ga - gb).max() / np.abs(ga).max()))
    assert worst < 1e-10, worst
