"""NumPy restatement of frcnn_optimizer_update: the WeightDecay hook and Chainer v1's update_one_cpu of MomentumSGD, Adam,
AdaGrad and RMSprop in float32, one rounding per operation in the order NumPy evaluates Chainer's expressions.  The
Python-float constants arrive already rounded to float32, in the hyper layout of include/frcnn_b200.h."""
import numpy as np

from backward_ref import fmaf

MOMENTUM_SGD, ADAM, ADAGRAD, RMSPROP = 0, 1, 2, 3
f32 = np.float32


def update(rule, w, s0, s1, g, hyper):
    """One update of float32 arrays; g is the (widened) gradient, hyper float32 [5].  Returns new (w, s0, s1)."""
    h = [f32(x) for x in hyper]
    w, s0 = w.astype(f32), s0.astype(f32)
    with np.errstate(all="ignore"):
        g = fmaf(np.full_like(w, h[0]), w, g.astype(f32))                       # WeightDecay: g += rate * w
        if rule == MOMENTUM_SGD:                                                # v *= momentum; v -= lr * g; w += v
            s0 = (h[2] * s0) - (h[1] * g)
            w = w + s0
        elif rule == ADAM:
            m, v = s0, s1.astype(f32)
            m = m + h[2] * (g - m)                                              # m += (1 - beta1) * (grad - m)
            v = v + h[3] * (g * g - v)                                          # v += (1 - beta2) * (grad * grad - v)
            w = w - (h[1] * m) / (np.sqrt(v) + h[4])                            # data -= lr * m / (sqrt(v) + eps)
            s0, s1 = m, v
        elif rule == ADAGRAD:
            s0 = s0 + g * g                                                     # h += grad * grad
            w = w - (h[1] * g) / (np.sqrt(s0) + h[2])                           # data -= lr * grad / (sqrt(h) + eps)
        else:
            s0 = s0 * h[2]                                                      # ms *= alpha
            s0 = s0 + (h[3] * g) * g                                            # ms += (1 - alpha) * grad * grad
            w = w - (h[1] * g) / (np.sqrt(s0) + h[4])                           # data -= lr * grad / (sqrt(ms) + eps)
    for a in (w, s0) + ((s1,) if rule == ADAM else ()):
        assert a.dtype == f32
    return w, s0, (s1 if rule == ADAM else None)


def update_f64(rule, w, s0, s1, g, rate, hp):
    """The same rule in float64 from the unrounded hyper-parameters hp (a dict of Python floats; Adam's "lr_t" given)."""
    d = np.float64
    w, s0, g = w.astype(d), s0.astype(d), g.astype(d)
    g = g + rate * w
    if rule == MOMENTUM_SGD:
        s0 = hp["momentum"] * s0 - hp["lr"] * g
        return w + s0, s0, None
    if rule == ADAM:
        m = s0 + (1 - hp["beta1"]) * (g - s0)
        v = s1.astype(d) + (1 - hp["beta2"]) * (g * g - s1.astype(d))
        return w - hp["lr_t"] * m / (np.sqrt(v) + hp["eps"]), m, v
    if rule == ADAGRAD:
        s0 = s0 + g * g
        return w - hp["lr"] * g / (np.sqrt(s0) + hp["eps"]), s0, None
    s0 = hp["alpha"] * s0 + (1 - hp["alpha"]) * g * g
    return w - hp["lr"] * g / (np.sqrt(s0) + hp["eps"]), s0, None
