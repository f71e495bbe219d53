"""fp64 restatements of the TF 1.13 optimizer updates that the fused update kernel implements for Adam and RMSProp
(tf.train.AdamOptimizer / RMSPropOptimizer as built by the reference's build_optimizer, helper/trainer.py:171-197).

TEST INFRASTRUCTURE ONLY, like the network oracle in oracle/tcr_oracle.py: the product path never imports it.  Each function
follows TF's ApplyAdam / ApplyRMSProp kernel (training_ops.cc) step for step on arrays of any (equal) shape.
"""
from __future__ import annotations

import numpy as np


def adam_update(params, m, v, grads, lr: float, beta1_power: float, beta2_power: float, beta1: float = 0.9,
                beta2: float = 0.999, epsilon: float = 1e-8):
    """One tf.train.AdamOptimizer step (ApplyAdam, TF 1.13 training_ops.cc) in fp64, step for step:
        alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power)
        m += (g - m)(1 - beta1);  v += (g^2 - v)(1 - beta2);  w -= (m * alpha) / (sqrt(v) + epsilon)
    then the finish op's beta1_power *= beta1, beta2_power *= beta2.  Arrays of any (equal) shape, e.g. the flat buffers;
    beta*_power are the values before the step.  Returns (params, m, v, beta1_power, beta2_power) after it."""
    f = np.float64
    w, m, v, g = (np.asarray(x, f) for x in (params, m, v, grads))
    alpha = f(lr) * np.sqrt(f(1.0) - f(beta2_power)) / (f(1.0) - f(beta1_power))
    m = m + (g - m) * (f(1.0) - f(beta1))
    v = v + (g * g - v) * (f(1.0) - f(beta2))
    w = w - (m * alpha) / (np.sqrt(v) + f(epsilon))
    return w, m, v, f(beta1_power) * f(beta1), f(beta2_power) * f(beta2)


def rmsprop_update(params, ms, mom, grads, lr: float, decay: float = 0.9, momentum: float = 0.0, epsilon: float = 1e-10):
    """One tf.train.RMSPropOptimizer step (ApplyRMSProp, centered=False, TF 1.13 training_ops.cc) in fp64, step for step:
        ms += (g^2 - ms)(1 - decay);  mom = mom * momentum + g * lr / sqrt(ms + epsilon);  w -= mom
    (TF 1.x initialises the `ms` slot to 1.0 and `mom` to 0).  Returns (params, ms, mom) after the step."""
    f = np.float64
    w, ms, mom, g = (np.asarray(x, f) for x in (params, ms, mom, grads))
    ms = ms + (g * g - ms) * (f(1.0) - f(decay))
    mom = mom * f(momentum) + (g * f(lr)) / np.sqrt(ms + f(epsilon))
    return w - mom, ms, mom
