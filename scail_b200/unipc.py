"""UniPC multistep flow solver (Zhao et al., NeurIPS 2023): an opt-in replacement for the sampler's Euler update.

This module owns the policy.  Every step still costs one CFG forward; the solver reuses the model outputs of earlier steps
so that it reaches a given ODE error in fewer steps than Euler.  Both the predictor (UniP) and the corrector (UniC) are the
bh2 variant with data prediction, in the rectified-flow parametrisation x = (1 - sigma) x0 + sigma eps:

  alpha = 1 - sigma, lambda(sigma) = log(alpha / sigma)  (-inf at sigma = 1, +inf at sigma = 0)
  g_i = u + s (c - u)           the guided velocity of step i from the CFG pair (u, c)
  m_i = x_i - sigma_i g_i       the data prediction, at the latent before correction

For a step from s (model output m0) to t, with older outputs m_{s_k} newest first:
  h = lambda_t - lambda_s, hh = -h, phi1 = B = expm1(hh), r_k = (lambda_{s_k} - lambda_s) / h, D_k = (m_{s_k} - m0) / r_k,
  R row i (i = 1..p) = [r_1^(i-1), ..., r_{p-1}^(i-1), 1], b_i = phi_(i) i! / B with phi_(1) = phi1 / hh - 1 and
  phi_(i+1) = phi_(i) / hh - 1 / (i+1)!.
  predictor, order p: x_t = (sigma_t / sigma_s) x - alpha_t phi1 m0 - alpha_t B sum_k rho_k D_k, with no sum at p = 1,
      rho = [0.5] at p = 2 and rho = solve(R[:2, :2], b[:2]) at p = 3;
  corrector, order q, new output m_t: x_t = (sigma_t / sigma_s) x_last - alpha_t phi1 m0
      - alpha_t B (sum_{k<q} rho_k D_k + rho_q (m_t - m0)), with rho = [0.5] at q = 1 and rho = solve(R, b) otherwise.

Step i of n: compute m_i; for i >= 1 correct x_last from sigma_{i-1} to sigma_i at the order q of the previous predictor
(the result is x_i); x_last <- x_i; predict x_{i+1} at order p_i = min(order, n - i, i + 1).  An older point at sigma = 1
(lambda = -inf) is never used: older points are taken newest first and taking them stops there, which lowers the
effective order.  At lambda_s = -inf, phi1 = B = -1; the last step has p = 1 and sigma_t = 0, so x_n = m_{n-1}.

Each step is therefore one linear combination of x_last, x, m_i and at most three older outputs.  step_coefficients()
composes it in fp64 from the sigma schedule; UniPC.step rounds each coefficient once to fp32 and runs ops.unipc_step_,
one fused pass over the latent.  The outputs live in `order` fp32 slots in rotation (m_j in slot j mod order), next to an
fp32 copy x_last: (order + 1) extra copies of the latent.  No default order or step count is chosen: what real weights
need is not measured here.
"""
import math
import numbers
from dataclasses import dataclass

import numpy as np
import torch

from . import ops


def check_order(order):
    """The solver order: an int in {1, 2, 3}.  Raises TypeError for bools and non-ints, ValueError for other ints."""
    if isinstance(order, bool) or not isinstance(order, numbers.Integral):
        raise TypeError(f"UniPC order must be an int in {{1, 2, 3}}, got {order!r}")
    if not 1 <= int(order) <= 3:
        raise ValueError(f"UniPC order must be 1, 2 or 3, got {order!r}")
    return int(order)


def check_schedule(sigmas):
    """A sigma schedule (tensor, array or sequence) -> a list of Python floats.  It must be 1-D with at least two points,
    finite and strictly decreasing, with sigma_0 <= 1 and sigma_n = 0."""
    s = np.asarray(sigmas.detach().cpu() if isinstance(sigmas, torch.Tensor) else sigmas, dtype=np.float64)
    if s.ndim != 1 or s.size < 2:
        raise ValueError(f"solver: the sigma schedule must be 1-D with at least 2 points, got shape {tuple(s.shape)}")
    if not np.all(np.isfinite(s)):
        raise ValueError("solver: the sigma schedule must be finite")
    if not np.all(np.diff(s) < 0):
        raise ValueError("solver: the sigma schedule must be strictly decreasing")
    if s[0] > 1.0 or s[-1] != 0.0:
        raise ValueError(f"solver: the sigma schedule must start at sigma_0 <= 1 and end at 0, got {s[0]!r} ... {s[-1]!r}")
    return [float(x) for x in s]


def _lam(sigma):
    """lambda = log(alpha / sigma), alpha = 1 - sigma."""
    if sigma == 1.0:
        return -math.inf
    if sigma == 0.0:
        return math.inf
    return math.log1p(-sigma) - math.log(sigma)


def _bh2(lam_s, lam_t, p):
    """(h, phi1, B, [b_1..b_p]) of a step from lambda_s to lambda_t."""
    h = lam_t - lam_s
    hh = -h
    phi1 = math.expm1(hh)
    B = phi1
    b, hk, fact = [], phi1 / hh - 1.0, 1.0
    for i in range(1, p + 1):
        b.append(hk * fact / B)
        fact *= i + 1
        hk = hk / hh - 1.0 / fact
    return h, phi1, B, b


def _update(sig, s, t, older, order, corrector):
    """One UniP / UniC update from sig[s] to sig[t], with older = the schedule indices of the older outputs, newest first,
    and `order` the nominal p or q.  -> (coefficient of the input latent, coefficient of m0, {index: coefficient of m_index}
    for the older outputs, coefficient of the new output m_t (corrector only))."""
    lam_s, lam_t = _lam(sig[s]), _lam(sig[t])
    used = []
    for j in older[:order - 1]:
        if sig[j] == 1.0:  # lambda = -inf: taking older points stops here
            break
        used.append(j)
    p = len(used) + 1
    h, phi1, B, b = _bh2(lam_s, lam_t, p)
    alpha_t = 1.0 - sig[t]
    r = [(_lam(sig[j]) - lam_s) / h for j in used]
    if corrector:
        if p == 1:
            rho = [0.5]
        else:
            R = np.array([[rk ** i for rk in r] + [1.0] for i in range(p)])
            rho = list(np.linalg.solve(R, np.array(b)))
    elif p == 1:
        rho = []
    elif p == 2:
        rho = [0.5]
    else:
        R = np.array([[rk ** i for rk in r] for i in range(p - 1)])
        rho = list(np.linalg.solve(R, np.array(b[:p - 1])))
    c_in = sig[t] / sig[s]
    c_m0 = -alpha_t * phi1
    c_old = {}
    for j, rk, rh in zip(used, r, rho):  # -alpha_t B rho_k (m_j - m0) / r_k
        c = -alpha_t * B * float(rh) / rk
        c_old[j] = c
        c_m0 -= c
    c_new = 0.0
    if corrector:  # -alpha_t B rho_q (m_t - m0)
        c_new = -alpha_t * B * float(rho[-1])
        c_m0 -= c_new
    return c_in, c_m0, c_old, c_new


def predictor_order(i, n, order):
    """The nominal order of step i's predictor (of n steps): min(order, n - i, i + 1)."""
    return min(order, n - i, i + 1)


@dataclass
class StepCoefficients:
    """Step i as the fused kernel computes it, in fp64.  m = x - sigma g; if `correct`, y = x_last_c * x_last + sum_k
    slot_c[k] * M_k + m_c * m, else y = x; then z = y_c * y + sum_k slot_p[k] * M_k + m_p * m.  M_k is slot k; the step
    writes m to slot `write`, y to x_last and z to x.  Slots absent from a step have coefficient exactly 0."""
    correct: bool
    x_last_c: float
    slot_c: list
    m_c: float
    y_c: float
    slot_p: list
    m_p: float
    write: int


def step_coefficients(sigmas, i, order):
    """The fp64 coefficients of step i of the schedule `sigmas` (a list of floats, as check_schedule returns it) at solver
    order `order`: pure host arithmetic, no GPU."""
    n = len(sigmas) - 1
    if not 0 <= i < n:
        raise ValueError(f"solver: step {i} is outside the schedule's {n} steps")
    slot_c, slot_p = [0.0] * order, [0.0] * order
    correct = i >= 1
    x_last_c = m_c = 0.0
    if correct:
        q = predictor_order(i - 1, n, order)
        # from sigma_{i-1} (m0 = m_{i-1}) to sigma_i, older outputs m_{i-2}, m_{i-3}, ..., new output m_i
        c_in, c_m0, c_old, m_c = _update(sigmas, i - 1, i, list(range(i - 2, -1, -1)), q, True)
        x_last_c = c_in
        slot_c[(i - 1) % order] += c_m0
        for j, c in c_old.items():
            slot_c[j % order] += c
    p = predictor_order(i, n, order)
    # from sigma_i (m0 = m_i, the new output) to sigma_{i+1}, older outputs m_{i-1}, m_{i-2}, ...
    y_c, m_p, c_old, _ = _update(sigmas, i, i + 1, list(range(i - 1, -1, -1)), p, False)
    for j, c in c_old.items():
        slot_p[j % order] += c
    return StepCoefficients(correct, x_last_c, slot_c, m_c, y_c, slot_p, m_p, i % order)


def _f32(c):
    return float(np.float32(c))


class UniPC:
    """UniPC multistep solver state of one sampling run, for sampler.sample / sampler_step / GraphedStep(solver=).

    order (1, 2 or 3): the highest order of the predictor; the corrector adds one.  begin(sigmas) binds a schedule (as
    sampler.make_flow_timesteps returns it) and drops all state; every step(x, v, scale, sigma, next_sigma) then has to be
    the next pair of that schedule, on the latent the state was built for at the first step."""

    def __init__(self, order=2):
        self._order = check_order(order)
        self._sigmas = None
        self.x_last = self.slots = self._buf_key = None
        self.reset()

    @property
    def order(self):
        return self._order

    @property
    def sigmas(self):
        return self._sigmas

    def begin(self, sigmas):
        """Bind a schedule (see check_schedule) and drop all state."""
        self._sigmas = check_schedule(sigmas)
        self.reset()

    def reset(self):
        """Drop the state (the next step is step 0 of the bound schedule).  The buffers are kept for a latent of the same
        shape: slots whose coefficient is 0 are never read, so nothing stale leaks into a new run."""
        self._i = 0
        self._key = None

    @property
    def step_index(self):
        return self._i

    def check_step(self, x, sigma, next_sigma):
        """Raise ValueError if step(x, ., ., sigma, next_sigma) cannot run now: no schedule bound, (sigma, next_sigma) not the
        next pair of it (compared as floats), or x not the latent the state was built for."""
        if self._sigmas is None:
            raise ValueError("solver: no sigma schedule is bound; call solver.begin(sigmas) first (sampler.sample does)")
        i, sig = self._i, self._sigmas
        if i >= len(sig) - 1:
            raise ValueError(f"solver: all {len(sig) - 1} steps of the bound schedule have run; call solver.begin(sigmas)")
        if float(sigma) != sig[i] or float(next_sigma) != sig[i + 1]:
            raise ValueError(f"solver: step {i} of the bound schedule goes from sigma {sig[i]!r} to {sig[i + 1]!r}, "
                             f"got ({float(sigma)!r}, {float(next_sigma)!r})")
        if i > 0 and self._key != (tuple(x.shape), x.dtype, x.device):
            raise ValueError(f"solver: the latent {tuple(x.shape)} {x.dtype} on {x.device} is not the latent "
                             f"{self._key[0]} {self._key[1]} on {self._key[2]} the solver's state was built for")

    def step(self, x, v, scale, sigma, next_sigma, delta=None, forecast=None, u_scale=None, m=None):
        """One solver step in place on x (fp32), from the CFG pair v (bf16 [2, ...], as cfg_euler_ reads it).  With `delta`
        (fp32, x's element count: a scail_b200.cfg_cache.CFGCache's held c - u), v is the conditional output alone (bf16
        [1, ...]) and u = f32(c) - delta; the coefficients and the state are those of the pair step.  `forecast` takes the
        place of delta for a CFGCache of order >= 1: (slots, coefficients), delta_hat = c0*S0 + c1*S1 + c2*S2 as
        ops.cfg_cache_delta_forecast forms it, and u = f32(c) - delta_hat.  u_scale (fp32 [1] on the device, from
        scail_b200.guidance.CFGZeroStar) scales u by s* before the guided combine.  With m (fp32, x's element count: the data
        prediction of scail_b200.guidance.APG), v and scale are not used and m takes the place of x - sigma*g; the coefficients,
        the slots and everything after m are the same.  Returns x."""
        if delta is not None and forecast is not None:
            raise ValueError("solver: pass delta or forecast, not both")
        if m is not None and (delta is not None or forecast is not None or u_scale is not None):
            raise ValueError("solver: a data prediction m takes no delta, forecast or u_scale")
        self.check_step(x, sigma, next_sigma)
        i = self._i
        if i == 0:
            key = (tuple(x.shape), x.dtype, x.device)
            if self._buf_key != key:
                self.x_last = self.slots = None  # free the old set before allocating the new one
                self.x_last = torch.empty_like(x)
                self.slots = torch.empty(self._order, x.numel(), device=x.device, dtype=torch.float32)
                self._buf_key = key
            self._key = key
        k = step_coefficients(self._sigmas, i, self._order)
        pad = [0.0] * (3 - self._order)
        coef = [k.x_last_c, *k.slot_c, *pad, k.m_c, k.y_c, *k.slot_p, *pad, k.m_p]
        coef = [_f32(c) for c in coef]
        kw = {} if u_scale is None else dict(u_scale=u_scale)
        if m is not None:
            ops.unipc_step_dpred_(x, self.x_last, m, self.slots, k.write, coef, k.correct)
        elif forecast is not None:
            ops.unipc_step_cached_forecast_(x, self.x_last, v, *forecast, self.slots, k.write, scale, self._sigmas[i], coef,
                                            k.correct, **kw)
        elif delta is None:
            ops.unipc_step_(x, self.x_last, v, self.slots, k.write, scale, self._sigmas[i], coef, k.correct, **kw)
        else:
            ops.unipc_step_cached_(x, self.x_last, v, delta, self.slots, k.write, scale, self._sigmas[i], coef, k.correct, **kw)
        self._i = i + 1
        return x
