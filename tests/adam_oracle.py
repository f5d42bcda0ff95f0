"""Float64 numpy restatements of the Adam block trainers of trainer/bmuf.py (reference) and of the Adam step they drive.

Test infrastructure only: the kernels (pika_b200/csrc/optim.cu) and the trainers (pika_b200/trainer/bmuf.py) are checked
against these.
"""
import numpy as np


def adam_step(p, g, m, v, lr, betas, eps, step):
    """torch.optim.Adam(lr, betas, eps, weight_decay=0, amsgrad=False).step() at ``step`` (the already-incremented count; it
    may be fractional after a BMUF-Adam sync).  Returns (p, m, v)."""
    b1, b2 = betas
    m = m + (1 - b1) * (g - m)
    v = b2 * v + (1 - b2) * g * g
    bc1 = 1 - b1 ** step
    bc2_sqrt = (1 - b2 ** step) ** 0.5
    return p - (lr / bc1) * m / (np.sqrt(v) / bc2_sqrt + eps), m, v


def clip_inf(g, max_norm):
    """clip_grad_norm_(g, max_norm, inf) in float32, as torch computes the coefficient: NaN anywhere gives a NaN coefficient"""
    g = np.asarray(g, np.float32)
    if max_norm <= 0:
        return g
    tot = np.float32(np.nan) if np.isnan(g).any() else np.float32(np.abs(g).max())
    coef = np.float32(max_norm) / (tot + np.float32(1e-6))
    coef = np.float32(np.nan) if np.isnan(coef) else min(coef, np.float32(1.0))
    return g * coef


def bmuf_adam_sync(glob, delta_prev, m_g, v_g, delta_sum, m_sum, v_sum, world, bm, blr, betas, tau, rho):
    """BmufAdamTrainer.update_and_sync's master update (trainer/bmuf.py:273-297) from the summed [delta; m; v]; ``rho`` is the
    value BEFORE this sync.  Returns (glob, delta_prev, m_g, v_g, rho); the local parameters and moments become glob, m_g, v_g,
    and the optimiser's step grows by rho_new * bm (:311)."""
    rho = bm * rho + tau
    d, ma, va = delta_sum / world, m_sum / world, v_sum / world
    delta_prev = bm * delta_prev + blr * (1 - bm) * d
    glob = glob - (1 + bm) * delta_prev
    (b1, b2) = betas
    b1t, b2t, b1r, b2r = b1 ** tau, b2 ** tau, b1 ** (rho * bm), b2 ** (rho * bm)
    m_g = (b1t * (b1r - 1) * m_g + (1 - b1t * b1r) * ma) / (1 - b1t)
    v_g = (b2t * (b2r - 1) * v_g + (1 - b2t * b2r) * va) / (1 - b2t)
    return glob, delta_prev, m_g, v_g, rho


def block_adam_sync(glob, m, v, step, delta_sum, block_lr, betas=(0.9, 0.999), eps=1e-8):
    """BlockAdamTrainer.update_and_sync (trainer/bmuf.py:146-168): Adam at block_lr on the SUMMED delta (not divided by the
    world size, :161).  ``step`` is the count before this sync.  Returns (glob, m, v, step); the local parameters become glob."""
    step = step + 1
    glob, m, v = adam_step(glob, delta_sum, m, v, block_lr, betas, eps, step)
    return glob, m, v, step
