"""GPU tests of the optimizer rules: frcnn_optimizer_update against the NumPy restatement (tests/optimizer_ref.py) bit for
bit, and the trainers' use of it.

- kernel: every rule with fp32 and bf16 gradients over several updates, n = 0, 1..9, 2^20+3 and unaligned slices, on
  zero, huge, subnormal, infinite and NaN inputs, with the hyper-parameters changed between updates; NaN compared as NaN
  whatever its payload.  MomentumSGD through the new entry equals frcnn_sgd_momentum and _bf16g bit for bit.
- trainers: a canvas trainer at N = 1 is bit-identical to its one-image trainer, so the eager trainer is the reference
  for the captured one.  For every rule the learning rate drops to a tenth after step 2 -- after the capture -- and
  w_flat and every state buffer must still agree after every step.  Then a ResNet-50 canvas trainer with Adam, a resume
  through optimizer_state / load_optimizer_state, and the drop-in trainer swap keeping Adam's m, v and t."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import optimizer_ref as oref

pytestmark = pytest.mark.gpu
DEV = "cuda"
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def _opt(rule, **kw):
    from frcnn_b200 import optimizers as O
    return O.RULES[rule](**kw)


def _bits_equal(got, want):
    """float32 arrays equal bit for bit; a NaN matches any NaN."""
    got, want = np.asarray(got, f32), np.asarray(want, f32)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.int32), want[~nan].view(np.int32))


def _flat_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------------ the kernel
SPECIAL = np.array([0.0, -0.0, 1e-40, -3e-42, 1.4e-45, 1.1754942e-38, 3e38, -3e38, 1e20, -1e19, np.inf, -np.inf, np.nan,
                    1.0, -2.5, 1e-20], f32)


def _data(n, rule, seed):
    rng = np.random.default_rng(seed)
    w = rng.standard_normal(n).astype(f32)
    s0 = (rng.standard_normal(n) * 0.01).astype(f32)
    s1 = np.abs(rng.standard_normal(n) * 1e-4).astype(f32)
    if rule in (oref.ADAGRAD, oref.RMSPROP):
        s0 = np.abs(s0)
    k = min(n, len(SPECIAL))
    if n >= 2:                                   # special weights and states at the front, shifted against the gradients
        w[:k] = np.roll(SPECIAL, 3)[:k]
        s0[:k] = np.abs(np.roll(SPECIAL, 5)[:k]) if rule in (oref.ADAGRAD, oref.RMSPROP) else np.roll(SPECIAL, 5)[:k]
    return w, s0, s1


def _grad(n, seed, t):
    rng = np.random.default_rng(seed * 31 + t)
    g = (rng.standard_normal(n) * 0.1).astype(f32)
    k = min(n, len(SPECIAL))
    g[:k] = np.roll(SPECIAL, t)[:k]
    if n > 64:
        g[-7:] = [0, 0, 1e-41, 3.3e38, np.nan, -1e-39, 2.0]
    return g


def _check_rule(rule, n, bf16, offset=0, steps=3, seed=1):
    """`steps` updates of an n-element slice starting `offset` elements into its buffers; after update 2 every
    hyper-parameter changes (the decay rate too).  Compares w and the state with the restatement after every update."""
    from frcnn_b200 import train_ops
    w, s0, s1 = _data(n, rule, seed)
    pad = lambda a: np.concatenate([np.full(offset, 7.0, f32), a])          # noqa: E731
    W, S0, S1 = (torch.from_numpy(pad(a)).to(DEV) for a in (w, s0, s1))
    wd, a_d, b_d = W[offset:], S0[offset:], (S1[offset:] if rule == oref.ADAM else None)
    hyper = torch.zeros(5, dtype=torch.float32, device=DEV)
    opt, rate = _opt(rule), 0.0005
    for t in range(1, steps + 1):
        if t == 3:
            rate = 0.01
            if rule == oref.MOMENTUM_SGD:
                opt.lr, opt.momentum = opt.lr * 0.1, 0.5
            elif rule == oref.ADAM:
                opt.alpha, opt.beta1, opt.beta2, opt.eps = opt.alpha * 0.1, 0.8, 0.99, 1e-6
            else:
                opt.lr, opt.eps = opt.lr * 0.1, 1e-6
                if rule == oref.RMSPROP:
                    opt.alpha = 0.9
        h = opt.hyper(rate, t)
        hyper.copy_(torch.from_numpy(h))
        G = torch.from_numpy(pad(_grad(n, seed, t))).to(DEV)
        if bf16:
            G = G.to(torch.bfloat16)
        g = G[offset:]
        train_ops.optimizer_update(rule, wd, a_d, b_d, g, hyper)
        w, s0, s1 = oref.update(rule, w, s0, s1, g.float().cpu().numpy(), h)
        torch.cuda.synchronize()
        assert _bits_equal(wd.cpu().numpy(), w), (rule, n, bf16, t, "w")
        assert _bits_equal(a_d.cpu().numpy(), s0), (rule, n, bf16, t, "s0")
        if rule == oref.ADAM:
            assert _bits_equal(b_d.cpu().numpy(), s1), (rule, n, bf16, t, "s1")
        assert (W[:offset] == 7).all() and (S0[:offset] == 7).all()


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("n", list(range(1, 10)) + [2 ** 20 + 3])
@pytest.mark.parametrize("rule", [0, 1, 2, 3])
def test_rule_bit_exact(rule, n, bf16):
    _check_rule(rule, n, bf16)


@pytest.mark.parametrize("offset,n", [(1, 1000), (3, 4099), (5, 33)])
@pytest.mark.parametrize("rule", [0, 1, 2, 3])
def test_rule_bit_exact_on_unaligned_slices(rule, offset, n):
    _check_rule(rule, n, rule % 2 == 1, offset=offset)


def test_inputs_reach_every_special_case():
    """The data puts a NaN, an infinity, a subnormal and a zero in each of w, s0 and g of the short runs."""
    w, s0, _ = _data(16, oref.ADAM, 1)
    g = _grad(16, 1, 1)
    for a in (w, s0, g):
        assert np.isnan(a).any() and np.isinf(a).any() and (a == 0).any() and ((a != 0) & (np.abs(a) < 1.1754944e-38)).any()


def test_no_elements():
    from frcnn_b200 import _lib
    from frcnn_b200.ops import _p, _stream
    lib = _lib.load()
    w, s0, s1, g = (torch.full((4,), x, device=DEV) for x in (1.0, 2.0, 3.0, 4.0))
    hyper = torch.ones(5, device=DEV)
    for rule in range(4):
        for bf in (0, 1):
            assert lib.frcnn_optimizer_update(rule, _p(w), _p(s0), _p(s1) if rule == 1 else None, _p(g), bf, 0, _p(hyper),
                                              _stream()) == 0
    torch.cuda.synchronize()
    assert (w == 1).all() and (s0 == 2).all() and (s1 == 3).all()


@pytest.mark.parametrize("bf16", [False, True])
def test_momentum_sgd_equals_the_existing_entries(bf16):
    from frcnn_b200 import train_ops
    n = 2 ** 20 + 3
    w, v, _ = _data(n, 0, 5)
    g = torch.from_numpy(_grad(n, 5, 1)).to(DEV)
    if bf16:
        g = g.to(torch.bfloat16)
    a_w, a_v, b_w, b_v = (torch.from_numpy(x.copy()).to(DEV) for x in (w, v, w, v))
    lr, mom, wd = 0.001, 0.9, 0.0005
    hyper = torch.from_numpy(_opt(0, lr=lr, momentum=mom).hyper(wd, 1)).to(DEV)
    train_ops.optimizer_update(0, a_w, a_v, None, g, hyper)
    getattr(train_ops, "sgd_momentum_bf16g" if bf16 else "sgd_momentum")(b_w, b_v, g, lr, mom, wd)
    torch.cuda.synchronize()
    assert _flat_equal(a_w, b_w) and _flat_equal(a_v, b_v)


# ------------------------------------------------------------------------------------------------ the trainers
_CACHE = {}


def _vgg_case():
    if "vgg" not in _CACHE:
        from test_canvas_rcnn_train_gpu import _rcnn_params
        from test_canvas_train_gpu import _images
        H, W = 296, 392
        _CACHE["vgg"] = (_rcnn_params(H, W, 3), _images([(H, W)] * 4, 4))
    return _CACHE["vgg"]


def _states_equal(a, b):
    return _flat_equal(a.w_flat, b.w_flat) and set(a.opt_state) == set(b.opt_state) and all(
        _flat_equal(a.opt_state[k], b.opt_state[k]) for k in a.opt_state)


def _drop_lr(tr):
    tr.lr = tr.lr * 0.1


RULE_KW = {1: dict(alpha=0.0005), 2: dict(lr=0.001), 3: dict(lr=0.0005)}


@pytest.mark.parametrize("rule", [0, 1, 2, 3])
def test_captured_rpn_step_follows_the_optimizer(rule):
    """CanvasRpnTrainer(N = 1) through step() -- eager, captured, replayed -- against RpnTrainer; the learning rate drops
    after step 2.  MomentumSGD is built from the lr keyword (the default optimizer) and dropped through trainer.lr."""
    from frcnn_b200.train_engine import CanvasRpnTrainer, RpnTrainer
    params, (xs, gts) = _vgg_case()
    H, W = xs[0].shape[1:]
    kw = dict(lr=0.001) if rule == 0 else dict(optimizer=_opt(rule, **RULE_KW[rule]))
    rt = RpnTrainer(params, H, W, ANCHORS, subsample="none", **kw)
    kw = dict(lr=0.001) if rule == 0 else dict(optimizer=_opt(rule, **RULE_KW[rule]))
    ct = CanvasRpnTrainer(params, 1, H, W, ANCHORS, subsample="none", **kw)
    for k in range(4):
        if k == 2:
            _drop_lr(rt)
            _drop_lr(ct)
        lr_ = rt.step(xs[k], gts[k])
        lc = ct.step([xs[k]], [gts[k]])
        torch.cuda.synchronize()
        assert ct.graph is not None
        assert _flat_equal(lc[0], lr_), k
        assert _states_equal(ct, rt), k
        assert ct.opt_t == rt.opt_t == k + 1


@pytest.mark.parametrize("rule", [0, 1, 2, 3])
def test_captured_rcnn_step_follows_the_optimizer(rule):
    """CanvasRcnnTrainer(N = 1, kept lists, explicit masks) through step() against RcnnTrainer; lr drops after step 2."""
    from frcnn_b200.train_engine import CanvasRcnnTrainer, RcnnTrainer
    from test_canvas_rcnn_train_gpu import _keep_and_masks
    from test_resnet_canvas_train_gpu import _images
    params, (xs, _) = _vgg_case()
    H, W = xs[0].shape[1:]
    xs, gts = _images([(H, W)] * 4, 4)             # boxes over 40-70 % of the image: some proposal overlaps one every step
    post_n = 120
    kw = dict(lr=0.001) if rule == 0 else dict(optimizer=_opt(rule, **RULE_KW[rule]))
    rt = RcnnTrainer(params, H, W, ANCHORS, post_n=post_n, **kw)
    kw = dict(lr=0.001) if rule == 0 else dict(optimizer=_opt(rule, **RULE_KW[rule]))
    ct = CanvasRcnnTrainer(params, 1, H, W, ANCHORS, post_n=post_n, sample="list", dropout="explicit", **kw)
    for k in range(4):
        if k == 2:
            _drop_lr(rt)
            _drop_lr(ct)
        keep, masks = _keep_and_masks(rt, xs[k], gts[k], post_n, 10 + k)
        lr_ = rt.step(xs[k], gts[k], keep_inds=keep, masks=masks)
        lc = ct.step([xs[k]], [gts[k]], keep_inds=[keep], masks=[masks])
        torch.cuda.synchronize()
        assert _flat_equal(lc[0], lr_), k
        assert _states_equal(ct, rt), k


def test_resnet50_canvas_trainer_with_adam():
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer, ResNetRpnTrainer
    from test_resnet_canvas_train_gpu import _images
    from test_resnet_train_gpu import _case
    H, W = 200, 264
    params = _case(50, H, W, 2)[0]
    xs, gts = _images([(H, W)] * 3, 4)
    rt = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, subsample="none", optimizer=_opt(1, alpha=0.0005))
    ct = CanvasResNetRpnTrainer(params, 1, H, W, ANCHORS, n_layers=50, subsample="none", optimizer=_opt(1, alpha=0.0005))
    for k in range(3):
        if k == 2:
            rt.optimizer.alpha *= 0.1
            ct.optimizer.alpha *= 0.1
        lr_ = rt.step(xs[k], gts[k])
        lc = ct.step([xs[k]], [gts[k]])
        torch.cuda.synchronize()
        assert _flat_equal(lc[0], lr_), k
        assert _states_equal(ct, rt), k
    assert float(ct.opt_state["v"].abs().max()) > 0


def test_resume_equals_an_uninterrupted_run():
    """2 steps, optimizer_state() and export_params() into a new trainer, 2 more steps == 4 steps, bit for bit (Adam, whose
    t enters lr_t, on the captured canvas step)."""
    from frcnn_b200.train_engine import CanvasRpnTrainer
    params, (xs, gts) = _vgg_case()
    H, W = xs[0].shape[1:]
    make = lambda p: CanvasRpnTrainer(p, 1, H, W, ANCHORS, subsample="none", optimizer=_opt(1, alpha=0.0005))   # noqa: E731
    a, b = make(params), make(params)
    for k in range(4):
        a.step([xs[k]], [gts[k]])
    for k in range(2):
        b.step([xs[k]], [gts[k]])
    state, learnt = b.optimizer_state(), b.export_params()
    assert state["t"] == 2
    del b
    c = make(dict(params, **learnt))
    c.load_optimizer_state(state)
    for k in range(2, 4):
        c.step([xs[k]], [gts[k]])
    torch.cuda.synchronize()
    assert c.opt_t == a.opt_t == 4
    assert _states_equal(c, a)


def test_dropin_trainer_swap_keeps_adams_state():
    from frcnn_b200 import dropin
    dropin.install()
    from chainer import Variable
    from frcnn_b200.train_engine import RcnnTrainer
    from models.faster_rcnn import FasterRCNN
    from models.vgg16 import VGG16Prev
    np.random.seed(11)
    model = FasterRCNN(trunk_class=VGG16Prev)
    rng = np.random.default_rng(2)
    for path, p in model.namedparams():
        if path in ("/RPN/rpn_cls_score/W", "/RPN/rpn_bbox_pred/W"):
            p.data[...] = (rng.standard_normal(p.data.shape) * 0.03).astype(f32)
    model._params_changed()
    model.rcnn_train = True
    H, W = 296, 392
    x = Variable(orc.make_image(H, W, seed=5))
    gt = Variable(np.array([[[20, 30, 150, 170, 3], [100, 20, 330, 240, 7], [200, 150, 280, 280, 1]]], f32))
    info = Variable(np.array([[H, W]], np.int32))
    np.random.seed(3)
    model(x, info, gt)
    old = model.rcnn_trainer
    pl = model.RPN.proposal_layer
    tr = RcnnTrainer(model.param_dict(), H, W, pl._anchors, precision=model.precision, feat_stride=model._feat_stride,
                     num_classes=model._num_classes, delta=float(model._rcnn_delta), post_n=pl._post_nms_top_n,
                     pre_n=pl._pre_nms_top_n, nms_thresh=pl._nms_thresh, min_size=pl._min_size, optimizer=_opt(1),
                     weight_decay=0.0)
    assert tr.index == old.index
    model.__dict__["rcnn_trainer"] = tr
    for s in range(2):
        np.random.seed(4 + s)
        model(x, info, gt)
        assert model.rcnn_trainer is tr
        tr.backward()
        tr.update()
    m, v = tr.opt_state["m"].clone(), tr.opt_state["v"].clone()
    assert float(v.abs().max()) > 0
    np.random.seed(6)
    model(Variable(orc.make_image(264, 360, seed=6)), Variable(np.array([[264, 360]], np.int32)), gt)
    tr2 = model.rcnn_trainer
    assert tr2 is not tr and tr2.optimizer is tr.optimizer and tr2.weight_decay == 0.0
    assert tr2.opt_t == 2 and tr2.v_flat is None
    assert _flat_equal(tr2.opt_state["m"], m) and _flat_equal(tr2.opt_state["v"], v)
