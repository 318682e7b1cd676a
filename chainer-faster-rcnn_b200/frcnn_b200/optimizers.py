"""The trainers' update rules: Chainer v1's MomentumSGD, Adam, AdaGrad and RMSprop, under Chainer's names and defaults.

Each object holds a rule's hyper-parameters as plain attributes.  A trainer takes one as `optimizer=` and reads its values
again before every update, so `trainer.optimizer.lr *= 0.1` between steps takes effect at the next one, captured steps
included.  The trainer applies its `weight_decay` hook to every rule, as Chainer applies hooks to any optimizer.

`hyper(rate, t)` turns the values into the float32 array frcnn_optimizer_update reads (include/frcnn_b200.h gives the
layout per rule); `states` names the rule's per-parameter float32 state, as Chainer names it.
"""
import math
import numbers

import numpy as np

from ._lib import FrcnnError

MOMENTUM_SGD, ADAM, ADAGRAD, RMSPROP = 0, 1, 2, 3         # FRCNN_OPT_*
HYPER_LEN = 5                                             # FRCNN_OPT_HYPER_LEN


class _Rule(object):
    rule = None
    states = ()
    lr_name = "lr"                  # the attribute trainer.lr reads and writes
    _unit = ()                      # attributes that must lie in [0, 1)

    def _values(self):
        return [(k, getattr(self, k)) for k in self._names]

    def check(self):
        """Raises FrcnnError unless every hyper-parameter is a finite real number in its range."""
        who = type(self).__name__
        for k, v in self._values():
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v):
                raise FrcnnError("%s: %s must be a finite number (got %r)" % (who, k, v))
            if v < 0 or (k in self._unit and v >= 1):
                raise FrcnnError("%s: %s must be in %s (got %r)" % (who, k, "[0, 1)" if k in self._unit else "[0, inf)", v))

    def hyper(self, rate, t):
        """float32 [HYPER_LEN]: the values of update t (1, 2, ...) with the decay rate `rate`, each rounded once to float32."""
        out = np.zeros((HYPER_LEN,), dtype=np.float32)
        vals = [float(rate)] + self._hyper(int(t))
        out[:len(vals)] = vals
        return out

    def __repr__(self):
        return "%s(%s)" % (type(self).__name__, ", ".join("%s=%r" % kv for kv in self._values()))


class MomentumSGD(_Rule):
    """v = momentum*v - lr*g; w += v."""
    rule, states, _names, _unit = MOMENTUM_SGD, ("v",), ("lr", "momentum"), ("momentum",)

    def __init__(self, lr=0.01, momentum=0.9):
        self.lr, self.momentum = lr, momentum

    def _hyper(self, t):
        return [float(self.lr), float(self.momentum)]


class Adam(_Rule):
    """m += (1-beta1)*(g-m); v += (1-beta2)*(g*g-v); w -= lr_t*m / (sqrt(v)+eps), lr_t = Chainer's Adam.lr at update t."""
    rule, states, lr_name = ADAM, ("m", "v"), "alpha"
    _names, _unit = ("alpha", "beta1", "beta2", "eps"), ("beta1", "beta2")

    def __init__(self, alpha=0.001, beta1=0.9, beta2=0.999, eps=1e-8):
        self.alpha, self.beta1, self.beta2, self.eps = alpha, beta1, beta2, eps

    def lr_t(self, t):
        """Chainer's Adam.lr at update t, in float64."""
        fix1 = 1. - math.pow(self.beta1, t)
        fix2 = 1. - math.pow(self.beta2, t)
        return self.alpha * math.sqrt(fix2) / fix1

    def _hyper(self, t):
        return [self.lr_t(t), 1. - self.beta1, 1. - self.beta2, float(self.eps)]


class AdaGrad(_Rule):
    """h += g*g; w -= lr*g / (sqrt(h)+eps)."""
    rule, states, _names = ADAGRAD, ("h",), ("lr", "eps")

    def __init__(self, lr=0.001, eps=1e-8):
        self.lr, self.eps = lr, eps

    def _hyper(self, t):
        return [float(self.lr), float(self.eps)]


class RMSprop(_Rule):
    """ms = alpha*ms + (1-alpha)*g*g; w -= lr*g / (sqrt(ms)+eps)."""
    rule, states, _names, _unit = RMSPROP, ("ms",), ("lr", "alpha", "eps"), ("alpha",)

    def __init__(self, lr=0.01, alpha=0.99, eps=1e-8):
        self.lr, self.alpha, self.eps = lr, alpha, eps

    def _hyper(self, t):
        return [float(self.lr), float(self.alpha), 1. - self.alpha, float(self.eps)]


RULES = (MomentumSGD, Adam, AdaGrad, RMSprop)


def resolve(optimizer, lr, momentum):
    """The trainer's rule: `optimizer` (checked), or MomentumSGD(lr, momentum) when it is None."""
    if optimizer is None:
        optimizer = MomentumSGD(lr=lr, momentum=momentum)
    if not isinstance(optimizer, RULES):
        raise FrcnnError("optimizer must be one of %s or None (got %r)" % (", ".join(r.__name__ for r in RULES), optimizer))
    optimizer.check()
    return optimizer
