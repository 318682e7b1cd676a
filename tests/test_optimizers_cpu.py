"""CPU tests of the optimizer rules: the frcnn_optimizer_update ABI (symbol, rule constants, argument types and errors), the
NumPy restatement against float64, the hyper-parameter objects, and the trainers' use of them on device="cpu" through
the launch recorder of test_trainer_launches_cpu (one update launch per step, one hyper array for the trainer's life, a
bad optimizer rejected before anything is allocated, state save and load)."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import optimizer_ref as oref
from test_train_targets_abi_cpu import _params
from test_trainer_launches_cpu import ANCHORS, H, W, Recorder, _canvas_rpn, _install, _rpn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p(256)
f32 = np.float32


@pytest.fixture
def rec(monkeypatch):
    from frcnn_b200 import _lib
    r = Recorder(_lib.load())
    _install(monkeypatch.setattr, r)
    return r


_PARAMS = {}


def _vgg_params():
    """One set of VGG16 parameters for the whole file (no test changes it)."""
    if not _PARAMS:
        import frcnn_oracle as orc
        _PARAMS.update(orc.make_params(seed=5))
    return _PARAMS


def _rules():
    from frcnn_b200 import optimizers as O
    return [O.MomentumSGD(lr=0.01, momentum=0.9), O.Adam(alpha=0.001), O.AdaGrad(lr=0.01), O.RMSprop(lr=0.01)]


# ------------------------------------------------------------------------------------------------ ABI
def test_abi_symbol_constants_and_types():
    from frcnn_b200 import _lib, optimizers as O
    lib = _lib.load()
    params = _params("frcnn_optimizer_update")
    assert params == ["int rule", "float* w", "float* s0", "float* s1", "const void* g", "int g_bf16", "long n",
                      "const float* hyper", "void* stream"]
    res, args = _lib.SIGNATURES["frcnn_optimizer_update"]
    assert res is ctypes.c_int and lib.frcnn_optimizer_update.argtypes == args
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long}
    for p, a in zip(params, args):
        typ = p.rsplit(" ", 1)[0].replace("const ", "")
        assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), p
    hdr = open(os.path.join(ROOT, "include", "frcnn_b200.h")).read()
    consts = dict((k, int(v)) for k, v in re.findall(r"#define FRCNN_OPT_(\w+) (\d+)", hdr))
    assert consts == dict(MOMENTUM_SGD=O.MOMENTUM_SGD, ADAM=O.ADAM, ADAGRAD=O.ADAGRAD, RMSPROP=O.RMSPROP,
                          HYPER_LEN=O.HYPER_LEN)
    assert [r.rule for r in O.RULES] == [0, 1, 2, 3]
    assert (O.MOMENTUM_SGD, O.ADAM, O.ADAGRAD, O.RMSPROP) == (oref.MOMENTUM_SGD, oref.ADAM, oref.ADAGRAD, oref.RMSPROP)


@pytest.mark.parametrize("bad,words", [
    (dict(rule=4), ["unknown rule 4"]), (dict(rule=-1), ["unknown rule -1"]), (dict(w=None), ["null pointer"]),
    (dict(s0=None), ["null pointer"]), (dict(g=None), ["null pointer"]), (dict(hyper=None), ["null pointer"]),
    (dict(rule=1), ["s1 must be given"]), (dict(s1=P), ["s1 must be NULL"]), (dict(rule=2, s1=P), ["s1 must be NULL"]),
    (dict(g_bf16=2), ["g_bf16 must be 0 or 1"]), (dict(n=-1), ["n = -1"])])
def test_argument_errors(bad, words):
    from frcnn_b200 import _lib
    lib = _lib.load()
    a = dict(rule=0, w=P, s0=P, s1=None, g=P, g_bf16=0, n=10, hyper=P)
    a.update(bad)
    st = lib.frcnn_optimizer_update(a["rule"], a["w"], a["s0"], a["s1"], a["g"], a["g_bf16"], a["n"], a["hyper"], None)
    assert st == _lib.ERR_ARG
    msg = _lib.last_error()
    assert "optimizer_update:" in msg and all(w in msg for w in words), msg


def test_no_elements_launches_nothing():
    from frcnn_b200 import _lib
    lib = _lib.load()
    for rule in range(4):
        assert lib.frcnn_optimizer_update(rule, P, P, P if rule == 1 else None, P, 1, 0, P, None) == _lib.OK


# ------------------------------------------------------------------------------------------------ the restatement
def _hand_picked():
    w = np.array([0.5, -1.25, 3.0, 1e-3, -7.5, 0.0, 2.0, -0.031], f32)
    g = np.array([0.1, 2.0, -0.75, 1e-4, 0.0, -3.0, 1.5e-2, 40.0], f32)
    s0 = np.array([0.0, 0.01, -0.2, 1e-6, 0.5, 0.0, 0.3, -1.0], f32)
    s1 = np.array([0.0, 0.25, 0.04, 1e-8, 2.0, 0.0, 9e-2, 1.0], f32)
    return w, g, s0, s1


@pytest.mark.parametrize("rule", [0, 1, 2, 3])
def test_restatement_agrees_with_float64(rule):
    """Over three updates the float32 restatement stays within a few float32 roundings of the float64 rule."""
    from frcnn_b200 import optimizers as O
    opt = _rules()[rule]
    w, g, s0, s1 = _hand_picked()
    if rule in (2, 3):
        s0 = np.abs(s0)
    rate = 0.0005
    W32, A32, B32 = w, s0, (s1 if rule == 1 else None)
    W64, A64, B64 = w.astype(np.float64), s0.astype(np.float64), (s1.astype(np.float64) if rule == 1 else None)
    for t in (1, 2, 3):
        hp = {k: float(getattr(opt, k)) for k in opt._names}
        if rule == 1:
            hp["lr_t"] = opt.lr_t(t)
        W32, A32, B32 = oref.update(rule, W32, A32, B32, g, opt.hyper(rate, t))
        W64, A64, B64 = oref.update_f64(rule, W64, A64, B64, g.astype(np.float64), rate, hp)
        for got, want, name in ((W32, W64, "w"), (A32, A64, "s0"), (B32, B64, "s1")):
            if want is None:
                continue
            scale = max(float(np.abs(want).max()), 1e-30)
            assert float(np.abs(got - want).max()) <= 16 * 2.0 ** -24 * scale, (O.RULES[rule].__name__, t, name)


def test_momentum_sgd_restatement_is_the_existing_one():
    import backward_ref as br
    w, g, s0, _ = _hand_picked()
    got = oref.update(0, w, s0, None, g, np.array([0.0005, 0.001, 0.9, 0, 0], f32))
    want = br.sgd_momentum(w, s0, g, 0.001, 0.9, 0.0005)
    assert np.array_equal(got[0].view(np.int32), want[0].view(np.int32))
    assert np.array_equal(got[1].view(np.int32), want[1].view(np.int32))


# ------------------------------------------------------------------------------------------------ the objects
def test_defaults_and_hyper_layout():
    from frcnn_b200 import optimizers as O
    assert (O.MomentumSGD().lr, O.MomentumSGD().momentum) == (0.01, 0.9)
    a = O.Adam()
    assert (a.alpha, a.beta1, a.beta2, a.eps) == (0.001, 0.9, 0.999, 1e-8)
    assert (O.AdaGrad().lr, O.AdaGrad().eps) == (0.001, 1e-8)
    r = O.RMSprop()
    assert (r.lr, r.alpha, r.eps) == (0.01, 0.99, 1e-8)
    assert O.MomentumSGD(0.02, 0.5).hyper(0.1, 7).tolist() == [f32(0.1), f32(0.02), f32(0.5), 0, 0]
    for t in (1, 2, 10, 1000):
        lr_t = 0.001 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        assert a.hyper(0.0005, t).tolist() == [f32(0.0005), f32(lr_t), f32(1 - 0.9), f32(1 - 0.999), f32(1e-8)]
    assert O.AdaGrad().hyper(0, 3).tolist() == [0, f32(0.001), f32(1e-8), 0, 0]
    assert r.hyper(0, 1).tolist() == [0, f32(0.01), f32(0.99), f32(1 - 0.99), f32(1e-8)]
    assert f32(1 - 0.99) != f32(1) - f32(0.99)           # the constant is rounded once, from float64


def _bad_optimizers():
    from frcnn_b200 import optimizers as O
    return ["adam", O.Adam, 0.01, O.MomentumSGD(lr=float("nan")), O.MomentumSGD(lr=-1e-3), O.MomentumSGD(momentum=1.0),
            O.Adam(beta1=1.0), O.Adam(beta2=-0.1), O.Adam(alpha="0.001"), O.Adam(eps=float("inf")), O.AdaGrad(eps=-1e-8),
            O.RMSprop(alpha=1.5), O.RMSprop(lr=True)]


@pytest.mark.parametrize("kind,k", [("rpn", k) for k in range(13)] + [("canvas_rpn", 0), ("canvas_rpn", 6), ("rcnn", 3),
                                                                      ("resnet_canvas_rcnn", 11)])
def test_bad_optimizer_is_rejected_before_allocation(monkeypatch, kind, k):
    from frcnn_b200 import train_engine
    from frcnn_b200._lib import FrcnnError

    def alloc(*a, **kw):
        raise AssertionError("the trainer allocated its buffers before it rejected the optimizer")
    monkeypatch.setattr(train_engine._ConvTrainer, "_init_params", alloc)
    bad = _bad_optimizers()[k]
    with pytest.raises(FrcnnError) as e:
        if kind == "resnet_canvas_rcnn":
            import frcnn_oracle as orc
            from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer
            CanvasResNetRcnnTrainer(orc.make_resnet_params(50, seed=3), 1, H, W, ANCHORS, n_layers=50, device="cpu",
                                    optimizer=bad)
        else:
            dict(rpn=_rpn, canvas_rpn=_canvas_rpn, rcnn=lambda p, **kw: _rcnn_opt(p, **kw))[kind](_vgg_params(), optimizer=bad)
    assert "optimizer" in str(e.value) or "must be" in str(e.value), str(e.value)


def _rcnn_opt(params, **kw):
    from frcnn_b200.train_engine import RcnnTrainer
    return RcnnTrainer(params, H, W, ANCHORS, post_n=64, sample="numpy", dropout=True, device="cpu", **kw)


# ------------------------------------------------------------------------------------------------ the trainers
@pytest.mark.parametrize("rule", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["rpn", "canvas_rpn"])
def test_update_launches_the_rule_once_with_one_hyper_array(rec, kind, rule):
    from frcnn_b200 import optimizers as O
    opt = _rules()[rule]
    tr = dict(rpn=_rpn, canvas_rpn=_canvas_rpn)[kind](_vgg_params(), optimizer=opt)
    assert sorted(tr.opt_state) == sorted(opt.states) and tr.optimizer is opt
    assert (tr.v_flat is tr.opt_state["v"]) if rule == O.MOMENTUM_SGD else tr.v_flat is None
    n = tr.w_flat.numel()
    hyper_ptrs = []
    for step in range(3):
        rec.reset()
        tr.update()
        calls = [c for c in rec.calls if c[0] == "frcnn_optimizer_update"]
        assert len(calls) == 1, [c[0] for c in rec.calls]
        assert [c[0] for c in rec.calls].count("frcnn_sgd_momentum") == 0
        _, r, w, s0, s1, g, g_bf16, nn, hyper, _ = calls[0]
        assert (r, g_bf16, nn) == (rule, 0, n) and (s1 is None) == (rule != O.ADAM)
        hyper_ptrs.append(tr.hyper.data_ptr())
        assert tr.opt_t == step + 1
        assert np.array_equal(tr.hyper.numpy(), opt.hyper(tr.weight_decay, step + 1))
        tr.lr = tr.lr * 0.1                                  # read at the next update
    assert len(set(hyper_ptrs)) == 1


def test_update_passes_the_trainer_buffers(rec):
    from frcnn_b200 import optimizers as O
    tr = _rpn(_vgg_params(), optimizer=O.Adam())
    rec.reset()
    tr.update()
    call = [c for c in rec.calls if c[0] == "frcnn_optimizer_update"][0]
    names = {"p%d" % rec._ptrs[t.data_ptr()]: k for k, t in (("w", tr.w_flat), ("m", tr.opt_state["m"]),
                                                              ("v", tr.opt_state["v"]), ("g", tr.g_flat), ("hyper", tr.hyper))}
    assert [names[a] for a in call[2:6] + call[8:9]] == ["w", "m", "v", "g", "hyper"]


def test_default_optimizer_is_momentum_sgd_from_the_keywords(rec):
    tr = _rpn(_vgg_params(), lr=0.003, momentum=0.8, weight_decay=0.001)
    assert type(tr.optimizer).__name__ == "MomentumSGD"
    assert (tr.lr, tr.momentum, tr.weight_decay) == (0.003, 0.8, 0.001)
    tr.lr, tr.momentum = 0.0003, 0.5
    assert (tr.optimizer.lr, tr.optimizer.momentum) == (0.0003, 0.5)


def test_lr_is_adams_alpha_and_momentum_is_momentum_sgds(rec):
    from frcnn_b200 import optimizers as O
    tr = _rpn(_vgg_params(), optimizer=O.Adam(alpha=0.002))
    assert tr.lr == 0.002
    tr.lr = 0.0002
    assert tr.optimizer.alpha == 0.0002
    with pytest.raises(AttributeError):
        tr.momentum


def test_a_bad_value_set_during_a_run_raises_before_the_update(rec):
    from frcnn_b200 import optimizers as O
    from frcnn_b200._lib import FrcnnError
    tr = _rpn(_vgg_params(), optimizer=O.RMSprop())
    tr.optimizer.alpha = 1.0
    rec.reset()
    with pytest.raises(FrcnnError):
        tr.update()
    assert rec.calls == [] and tr.opt_t == 0


def test_optimizer_state_round_trip_in_reference_layout(rec):
    """optimizer_state() holds every trained parameter in the reference's layout (fc6/W in (c, h, w) columns, as
    export_params), and load_optimizer_state() puts it back into the flat buffers bit for bit."""
    from frcnn_b200 import optimizers as O
    from frcnn_b200._lib import FrcnnError
    a = _rcnn_opt(_vgg_params(), optimizer=O.Adam())
    g = torch.Generator().manual_seed(3)
    for buf in a.opt_state.values():
        buf.copy_(torch.randn(buf.shape, generator=g))
    a.opt_t = 7
    st = a.optimizer_state()
    assert st["rule"] == "Adam" and st["t"] == 7 and set(st) == {"rule", "t", "m", "v"}
    assert set(st["m"]) == set(a.index)
    # fc6/W uses export_params' layout: the same permutation of the flat buffer
    saved = a.w_flat.clone()
    a.w_flat.copy_(a.opt_state["m"])
    assert np.array_equal(a.export_params()["fc6/W"], st["m"]["fc6/W"])
    a.w_flat.copy_(saved)
    b = _rcnn_opt(_vgg_params(), optimizer=O.Adam())
    b.load_optimizer_state(st)
    assert b.opt_t == 7
    for k in ("m", "v"):
        assert torch.equal(b.opt_state[k].view(torch.int32), a.opt_state[k].view(torch.int32)), k
    dev = a.optimizer_state(to_host=False)
    c = _rcnn_opt(_vgg_params(), optimizer=O.Adam())
    c.load_optimizer_state(dev)
    assert torch.equal(c.opt_state["v"], a.opt_state["v"])
    with pytest.raises(FrcnnError):
        _rcnn_opt(_vgg_params()).load_optimizer_state(st)                     # MomentumSGD cannot load Adam's state
    st["m"].pop("fc7/b")
    with pytest.raises(FrcnnError):
        b.load_optimizer_state(st)
