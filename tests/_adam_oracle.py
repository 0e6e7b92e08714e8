"""numpy restatements of the fused Adam update (DESIGN.md section 21).

Update number t (t = 1 for the first) of every element, with g' = coef * g the clipped gradient:
    host, in double, each rounded once to fp32:
        step_size = lr / (1 - b1^t),  bc2s = sqrt(1 - b2^t),  omb1 = 1 - b1,  omb2 = 1 - b2
    device, fp32, each operation rounded on its own in this order:
        m = b1 * m + omb1 * g'
        v = b2 * v + omb2 * (g' * g')
        denom = sqrt(v) / bc2s + eps
        p = p - step_size * (m / denom)
`adam_fp32` is that, bit for bit (numpy float32 arithmetic contracts nothing; its sqrt and division are correctly
rounded).  `adam_fp64` is the same rule in float64 with exact scalars: the reference of the end-to-end checks.
"""
import numpy as np

f32 = np.float32


def scalars(lr, beta1, beta2, eps, t):
    """(b1, b2, omb1, omb2, eps, step_size, bc2s) of update t as the host computes them: fp32, rounded once from double."""
    b1, b2 = float(f32(beta1)), float(f32(beta2))
    return (f32(b1), f32(b2), f32(1.0 - b1), f32(1.0 - b2), f32(eps), f32(float(f32(lr)) / (1.0 - b1 ** t)),
            f32(np.sqrt(1.0 - b2 ** t)))


def adam_fp32(p, g, m, v, coef, lr, beta1, beta2, eps, t):
    """Update t in fp32: returns (p, g', m, v) as new float32 arrays."""
    b1, b2, omb1, omb2, e, step_size, bc2s = scalars(lr, beta1, beta2, eps, t)
    p, g, m, v = (np.asarray(a, dtype=f32) for a in (p, g, m, v))
    gs = g * f32(coef)
    m = b1 * m + omb1 * gs
    v = b2 * v + omb2 * (gs * gs)
    denom = np.sqrt(v) / bc2s + e
    p = p - step_size * (m / denom)
    return p, gs, m, v


def adam_fp64(p, g, m, v, coef, lr, beta1, beta2, eps, t):
    """Update t in float64 with exact scalars: returns (p, g', m, v)."""
    p, g, m, v = (np.asarray(a, dtype=np.float64) for a in (p, g, m, v))
    gs = g * coef
    m = beta1 * m + (1.0 - beta1) * gs
    v = beta2 * v + (1.0 - beta2) * gs * gs
    denom = np.sqrt(v) / np.sqrt(1.0 - beta2 ** t) + eps
    p = p - lr / (1.0 - beta1 ** t) * (m / denom)
    return p, gs, m, v
