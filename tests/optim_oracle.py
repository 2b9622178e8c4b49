"""fp32 numpy restatements of the 32-bit Lion, RMSprop and AdEMAMix updates, in the operation order of
`qlora_b200/csrc/optim32.cu` (upstream bitsandbytes' kOptimizer32bit1State LION / RMSPROP and kOptimizer32bit2State
ADEMAMIX), next to `oracle.nf4_oracle.adamw32bit_step`.  Every numpy operation on fp32 arrays is one correctly rounded
fp32 operation, as every operation of the kernel is.  Test infrastructure only."""
from __future__ import annotations

import math

import numpy as np


def lion32bit_step(p, g, m, lr, beta1, beta2, weight_decay, gnorm_scale=1.0):
    """Upstream's 32-bit 1-state LION update (kOptimizer32bit1State) restated in fp32 numpy, in the kernel's operation
    order; sign(0) = 0.  Returns (p_new, m_new) as fp32."""
    f = np.float32
    p, g, m = (np.asarray(a, dtype=np.float32) for a in (p, g, m))
    gi = f(gnorm_scale) * g
    c = f(beta1) * m + f(f(1.0) - f(beta1)) * gi
    if weight_decay > 0:
        p = p * f(f(1.0) - f(f(lr) * f(weight_decay)))
    p2 = p - f(lr) * np.sign(c).astype(np.float32)
    m2 = f(beta2) * m + f(f(1.0) - f(beta2)) * gi
    return p2.astype(np.float32), m2.astype(np.float32)


def rmsprop32bit_step(p, g, v, lr, alpha, eps, weight_decay, gnorm_scale=1.0):
    """Upstream's 32-bit 1-state RMSPROP update (kOptimizer32bit1State; no momentum, not centered) restated in fp32 numpy.
    Returns (p_new, v_new) as fp32."""
    f = np.float32
    p, g, v = (np.asarray(a, dtype=np.float32) for a in (p, g, v))
    gi = f(gnorm_scale) * g
    if weight_decay > 0:
        gi = gi + f(weight_decay) * p
    v2 = f(alpha) * v + f(f(1.0) - f(alpha)) * (gi * gi)
    p2 = p - f(lr) * (gi / (np.sqrt(v2) + f(eps)))
    return p2.astype(np.float32), v2.astype(np.float32)


def ademamix_step_scalars(step, beta1, beta2, beta3, alpha, t_alpha=None, t_beta3=None):
    """AdEMAMix's per-step scalars (c1, c2, alpha_t, beta3_t): float64 from the fp32 hyper-parameters, rounded to fp32."""
    f = np.float32
    b1, b2, b3, al = (float(f(x)) for x in (beta1, beta2, beta3, alpha))
    t = float(step)
    c1 = f(1.0 - b1 ** t)
    c2 = f(math.sqrt(1.0 - b2 ** t))
    alpha_t = f(al) if not t_alpha else f(min(t * al / float(f(t_alpha)), al))
    if not t_beta3:
        beta3_t = f(b3)
    else:
        lb1, lb3, fr = math.log(b1), math.log(b3), t / float(f(t_beta3))
        beta3_t = f(min(math.exp(lb1 * lb3 / ((1.0 - fr) * lb3 + fr * lb1)), b3))
    return c1, c2, alpha_t, beta3_t


def ademamix32bit_step(p, g, m1, m2, nu, lr, beta1, beta2, beta3, alpha, eps, weight_decay, step, t_alpha=None, t_beta3=None,
                       gnorm_scale=1.0):
    """Upstream's 32-bit ADEMAMIX update (kOptimizer32bit2State) restated in fp32 numpy.  Returns (p, m1, m2, nu) as fp32."""
    f = np.float32
    p, g, m1, m2, nu = (np.asarray(a, dtype=np.float32) for a in (p, g, m1, m2, nu))
    c1, c2, alpha_t, beta3_t = ademamix_step_scalars(step, beta1, beta2, beta3, alpha, t_alpha, t_beta3)
    gi = f(gnorm_scale) * g
    m1 = f(beta1) * m1 + f(f(1.0) - f(beta1)) * gi
    m2 = beta3_t * m2 + f(f(1.0) - beta3_t) * gi
    nu = f(beta2) * nu + f(f(1.0) - f(beta2)) * (gi * gi)
    p2 = p - f(lr) * ((m1 / c1 + alpha_t * m2) / (np.sqrt(nu) / c2 + f(eps)))
    if weight_decay > 0:
        p2 = p2 * f(f(1.0) - f(f(lr) * f(weight_decay)))
    return p2.astype(np.float32), m1.astype(np.float32), m2.astype(np.float32), nu.astype(np.float32)
