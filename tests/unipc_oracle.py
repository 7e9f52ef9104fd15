"""fp64 restatement of the UniPC flow solver (bh2, data prediction), written from the formulas in scail_b200/unipc.py's
docstring: it keeps the model outputs, builds R and b and solves for rho at every predictor and corrector, and applies
the updates to the latent as written.  It does not use the product's composed coefficients."""
import math

import numpy as np


def lam(sigma):
    """lambda = log(alpha / sigma), alpha = 1 - sigma: -inf at sigma = 1, +inf at sigma = 0."""
    with np.errstate(divide="ignore"):
        return float(np.log(np.float64(1.0 - sigma)) - np.log(np.float64(sigma)))


def bh2_update(x, m0, sig_s, sig_t, older, order, m_t=None):
    """One UniP (m_t None) or UniC update of x from sig_s (model output m0) to sig_t.  older: [(sigma_k, m_k)] newest first.
    Older points at sigma = 1 are never used: taking them stops at the first one, which lowers the effective order."""
    use = []
    for s_k, m_k in older[:order - 1]:
        if s_k == 1.0:
            break
        use.append((s_k, m_k))
    p = len(use) + 1
    lam_s, lam_t = lam(sig_s), lam(sig_t)
    h = lam_t - lam_s
    hh = -h
    phi1 = math.expm1(hh)
    B = math.expm1(hh)
    alpha_t = 1.0 - sig_t
    rks, D = [], []
    for s_k, m_k in use:
        r = (lam(s_k) - lam_s) / h
        rks.append(r)
        D.append((m_k - m0) / r)
    rks.append(1.0)
    rks = np.array(rks)
    R, b = [], []
    phi_k = phi1 / hh - 1.0
    fact = 1
    for i in range(1, p + 1):
        R.append(rks ** (i - 1))
        b.append(phi_k * fact / B)
        fact *= i + 1
        phi_k = phi_k / hh - 1.0 / fact
    R, b = np.stack(R), np.array(b)
    base = (sig_t / sig_s) * x - alpha_t * phi1 * m0
    if m_t is None:  # predictor
        if p == 1:
            return base
        rho = np.array([0.5]) if p == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
        res = sum(rho[k] * D[k] for k in range(p - 1))
        return base - alpha_t * B * res
    rho = np.array([0.5]) if p == 1 else np.linalg.solve(R, b)  # corrector
    res = sum((rho[k] * D[k] for k in range(p - 1)), np.zeros_like(x))
    return base - alpha_t * B * (res + rho[-1] * (m_t - m0))


def sample(x, sigmas, order, velocity):
    """The whole solver in fp64.  x: the starting latent (ndarray), sigmas: the schedule, velocity(x, sigma, i) -> the guided
    velocity g_i (ndarray) at the latent before correction.  Returns the final latent."""
    sig = [float(s) for s in sigmas]
    n = len(sig) - 1
    x = np.asarray(x, dtype=np.float64).copy()
    ms, x_last, p_prev = [], None, None
    for i in range(n):
        m = x - sig[i] * np.asarray(velocity(x, sig[i], i), dtype=np.float64)
        if i >= 1:
            older = [(sig[i - 1 - k], ms[-1 - k]) for k in range(1, len(ms))]
            x = bh2_update(x_last, ms[-1], sig[i - 1], sig[i], older, p_prev, m_t=m)
        ms.append(m)
        x_last = x
        p = min(order, n - i, i + 1)
        older = [(sig[i - k], ms[-1 - k]) for k in range(1, len(ms))]
        x = bh2_update(x, m, sig[i], sig[i + 1], older, p)
        p_prev = p
    return x


def euler(x, sigmas, velocity):
    sig = [float(s) for s in sigmas]
    x = np.asarray(x, dtype=np.float64).copy()
    for i in range(len(sig) - 1):
        x = x + (sig[i + 1] - sig[i]) * np.asarray(velocity(x, sig[i], i), dtype=np.float64)
    return x


def gaussian_velocity(mu, s):
    """The exact velocity of x = (1 - sigma) x0 + sigma eps with x0 ~ N(mu, s^2) per element; from x = eps at sigma = 1 the
    ODE ends at mu + s eps."""
    def v(x, sigma, i=None):
        a = 1.0 - sigma
        return -mu + (x - a * mu) * (sigma - a * s * s) / (a * a * s * s + sigma * sigma)
    return v
