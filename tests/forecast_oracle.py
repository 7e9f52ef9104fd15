"""Test-side restatement of the first-block cache's Taylor forecast (FirstBlockCache(order >= 1)): the Lagrange coefficients
in fp64, the forecast kernels as separate torch fp32 elementwise ops, and whole cached forwards built from the model's own
hooks (patch embedding, layer_forward, final_forward).  The order-0 pieces come from tests/step_cache_oracle.py."""
import math

import numpy as np
import torch

from step_cache_oracle import indicator_sums, update_ref


def lagrange_coefficients(points, sigma):
    """points: [(sigma_i, tag_i)] newest first.  Drop the oldest points until the sigmas are pairwise distinct, then
    -> [(tag_i, c_i)] with c_i = prod_{k != i} (sigma - sigma_k) / (sigma_i - sigma_k) in fp64, rounded once to fp32."""
    m = len(points) - 1
    while m > 0 and len({s for s, _ in points[:m + 1]}) < m + 1:
        m -= 1
    used = points[:m + 1]
    out = []
    for si, tag in used:
        c = 1.0
        for sk, _ in used:
            if sk != si:
                c *= (sigma - sk) / (si - sk)
        out.append((tag, float(np.float32(c))))
    return out


def forecast_sum(R_slots, coef):
    """t = c0*R0, t = t + c1*R1, t = t + c2*R2 over the slots with c != 0, in slot order, one fp32 torch op per product and
    per sum (None when no slot is active)."""
    t = None
    for s, c in enumerate(coef):
        if c == 0.0:
            continue
        p = R_slots[s] * torch.tensor(c, dtype=torch.float32, device=R_slots.device)
        t = p if t is None else t + p
    return t


def apply_forecast_ref(h, R_slots, coef, n_ref):
    """h with its noise rows replaced by bf16(f32(h) + t), t = forecast_sum(R_slots, coef)."""
    out = h.clone()
    t = forecast_sum(R_slots, coef)
    if t is None:
        return out
    rows = out[:, n_ref:n_ref + R_slots.shape[2]]
    rows.copy_((rows.float() + t).to(torch.bfloat16))
    return out


class RestatedForecastCache:
    """The forecasting cache over whole forwards: forward(threshold, sigma, x, **model kwargs) -> the velocity, with
    history = [(indicator, skipped)] as FirstBlockCache keeps it."""

    def __init__(self, model, order, max_skips=None):
        self.m, self.order, self.max_skips = model, order, max_skips
        self.r_ref = None
        self.slots = None  # order + 1 fp32 residuals, zero at allocation
        self.slot_sigma = [None] * (order + 1)
        self.n_computed = 0
        self.run = 0
        self.history = []

    def forward(self, threshold, sigma, x, timesteps=None, context=None, **kwargs):
        m = self.m
        ad, fl = m.mixins["adaln_layer"], m.mixins["final_layer"]
        h0, kw, _ = m._tokens(x, timesteps, context, None, dict(kwargs))
        h0 = h0.clone()
        h1 = ad.layer_forward(h0.clone(), None, layer_id=0, **kw).clone()
        n_ref, n_seq = kw["ref_length"], kw["seq_length"]
        if self.slots is None:
            self.slots = torch.zeros(self.order + 1, h1.shape[0], n_seq, h1.shape[2], device=h1.device)
        r, num, den = indicator_sums(h0, h1, self.r_ref if self.r_ref is not None else torch.zeros_like(h1))
        ind = math.inf if den == 0 else num / den
        skip = self.r_ref is not None and ind < threshold and (self.max_skips is None or self.run < self.max_skips)
        self.run = self.run + 1 if skip else 0
        self.history.append((ind, skip))
        n = self.order + 1
        if skip:
            recent = [(self.n_computed - 1 - k) % n for k in range(min(n, self.n_computed))]
            coef = [0.0] * n
            for s, c in lagrange_coefficients([(self.slot_sigma[s], s) for s in recent], float(sigma)):
                coef[s] = c
            h = apply_forecast_ref(h1, self.slots, coef, n_ref)
        else:
            h = h1.clone()
            for l in range(1, m.num_layers):
                h = ad.layer_forward(h, None, layer_id=l, **kw)
            s = self.n_computed % n
            self.slots[s] = update_ref(h, h1[:, n_ref:n_ref + n_seq], n_ref)
            self.slot_sigma[s] = float(sigma)
            self.n_computed += 1
            self.r_ref = r
        return fl.final_forward(h, **kw)
