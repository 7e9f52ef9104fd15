"""First-block residual cache: skip DiT blocks 1..L-1 on sampler steps where block 0's residual has barely changed.

This module owns the policy.  Per forward of the CFG batch (both branches together):

  1. h0 = patch embedding; block 0 runs on a copy of it -> h1.
  2. r = bf16(h1 - h0) (computed in fp32, then rounded); ind = sum|r - r_ref| / sum|r_ref| over all B*N*d elements, where
     r_ref is r of the last COMPUTED step; a zero denominator gives +inf.
  3. Skip iff the cache holds state for this geometry and ind < threshold (a NaN never skips).  A skipped step feeds
     bf16(f32(h1) + R) on the noise rows to the final layer and updates nothing, so drift accumulates against the last
     computed step.
  4. Otherwise blocks 1..L-1 run as usual, then R = f32(h_L) - f32(h1) on the noise rows and r_ref <- r (a buffer swap).

The kernels are ops.step_cache_indicator / step_cache_update / step_cache_apply; DiffusionTransformer.forward(_step_cache=)
and sampler.sample / sampler_step / GraphedStep(step_cache=) drive them.  No default threshold is chosen: that needs real
weights and a visual check.

Taylor forecast (order >= 1).  Instead of holding R from the last computed step, the cache keeps the residuals of the last
order + 1 computed steps, each with the sampler's sigma of its step, in order + 1 fp32 slots (the j-th computed step since
reset() writes slot j mod (order + 1)).  A skipped step at sigma applies the Lagrange polynomial through the m + 1 most
recent (sigma_i, R_i), evaluated at sigma, where m = min(order, computed - 1), reduced further until those sigmas are
pairwise distinct.  The coefficients c_i = prod_{k != i} (sigma - sigma_k) / (sigma_i - sigma_k) are computed in fp64 on
the host and rounded once to fp32; unused slots get exactly 0 (the kernel then does not read them).  The skip decision is
the one above.  Each extra order costs one more slot: +0.88 GB at 512x512 and +1.54 GB at 512x896 (b = 2).  max_skips
caps the run of consecutive skipped steps, at every order.  The kernels are ops.step_cache_update_slot /
step_cache_apply_forecast; they read the slot index and the coefficients from a small device tensor (the control block),
which the host writes once per step between the skip decision and the blocks' tail.
"""
import math
import numbers

import numpy as np
import torch

from . import ops


def check_threshold(threshold, what="step cache"):
    """A float >= 0 (inf allowed).  Raises TypeError for bools and non-numbers, ValueError for NaN and negatives; the
    messages name `what`."""
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real):
        raise TypeError(f"{what} threshold must be a real number >= 0 (inf allowed), got {threshold!r}")
    t = float(threshold)
    if math.isnan(t) or t < 0:
        raise ValueError(f"{what} threshold must be >= 0 (inf allowed), got {threshold!r}")
    return t


def check_order(order, what="step cache"):
    """The degree of the forecast polynomial: an int in {0, 1, 2}.  Raises TypeError for bools and non-ints, ValueError for
    other ints; the messages name `what`."""
    if isinstance(order, bool) or not isinstance(order, numbers.Integral):
        raise TypeError(f"{what} order must be an int in {{0, 1, 2}}, got {order!r}")
    if not 0 <= int(order) <= 2:
        raise ValueError(f"{what} order must be 0, 1 or 2, got {order!r}")
    return int(order)


def check_max_skips(max_skips, what="step cache"):
    """None (no cap) or an int >= 0.  Raises TypeError for bools and non-ints, ValueError for negatives; the messages name
    `what`."""
    if max_skips is None:
        return None
    if isinstance(max_skips, bool) or not isinstance(max_skips, numbers.Integral):
        raise TypeError(f"{what} max_skips must be None or an int >= 0, got {max_skips!r}")
    if int(max_skips) < 0:
        raise ValueError(f"{what} max_skips must be None or an int >= 0, got {max_skips!r}")
    return int(max_skips)


def check_sigma(sigma, what="step cache"):
    """The sampler's sigma of a step as a finite float (a Python number or a one-element tensor, as sampler_step takes it);
    the messages name `what`."""
    if isinstance(sigma, bool):
        raise TypeError(f"{what} sigma must be a real number, got {sigma!r}")
    s = float(sigma)
    if not math.isfinite(s):
        raise ValueError(f"{what} sigma must be finite, got {sigma!r}")
    return s


def forecast_coefficients(sigma, slot_sigmas, n_computed, order):
    """The forecast of a skipped step at `sigma` -> the fp32 coefficient of each of the order + 1 slots (a list of Python
    floats, each exactly an fp32 value).  slot_sigmas[s] is the sigma of the computed step slot s holds; the j-th computed
    step (j = 0, 1, ...) went to slot j mod (order + 1), and n_computed steps have been computed.  The polynomial goes
    through the m + 1 most recent computed steps, m = min(order, n_computed - 1), with m reduced until their sigmas are
    pairwise distinct.  c_i = prod_{k != i} (sigma - sigma_k) / (sigma_i - sigma_k) in fp64, rounded once to fp32; the other
    slots get exactly 0."""
    n = order + 1
    coef = [0.0] * n
    if n_computed < 1:
        return coef
    m = min(order, n_computed - 1)
    recent = [(n_computed - 1 - k) % n for k in range(m + 1)]  # newest first
    while m > 0 and len({slot_sigmas[s] for s in recent[:m + 1]}) < m + 1:
        m -= 1
    used = recent[:m + 1]
    for i in used:
        c = 1.0
        for k in used:
            if k != i:
                c *= (sigma - slot_sigmas[k]) / (slot_sigmas[i] - slot_sigmas[k])
        coef[i] = float(np.float32(c))
    return coef


def indicator(num, den):
    """sum|r - r_ref| / sum|r_ref| from the two sums: +inf when the denominator is zero, NaN stays NaN (what the kernel's
    ratio computes)."""
    return math.inf if den == 0 else num / den


def check_supported(cp=None, chunk_dim=None, num_layers=None, plan=None):
    """Refuse the configurations the cache does not cover: every rank would have to agree on the skip decision (an
    all-reduce of the indicator) under context parallelism or a hybrid CFG plan, and a truncated or pre-chunked forward is
    not a full step."""
    if cp is not None and getattr(cp, "size", 1) > 1:
        raise NotImplementedError(f"step_cache is not implemented under context parallelism (a ContextParallel of size {cp.size}); "
                                  "run without a step cache or on one GPU")
    if plan is not None:
        raise NotImplementedError("step_cache is not implemented with a HybridParallel plan; run without a step cache or on one GPU")
    if chunk_dim is not None:
        raise NotImplementedError("step_cache is not implemented with chunk_dim (pre-chunked sequence parallelism)")
    if num_layers is not None:
        raise NotImplementedError("step_cache is not implemented with _num_layers: the cache needs the full stack of blocks")


class Buffers:
    """The cache's workspace for one geometry key (B, N, d, n_ref, n_seq, device): the working copy h1 that blocks 0..L-1
    run on, r_ref / r_new (bf16 [B, N, d]; r_ref starts at zero, so the first indicator is +inf), h1c (the noise rows of
    h1, bf16) and R (fp32 [B, n_seq, d]), plus the indicator's partial sums and its fp64 result {num, den, ratio, 0}.
    At order >= 1, R is None and R_slots (fp32 [order + 1, B, n_seq, d], zero-filled) takes its place, with slot_sigma (the
    sigma of the computed step each slot holds, None while empty), n_computed (computed steps written since allocation) and
    the control block ctl (int32 [4] on the device: the slot the next update writes, then the bits of the three fp32
    forecast coefficients), which write_control() fills once per step."""

    def __init__(self, key, order=0):
        B, N, d, n_ref, n_seq, device = key
        self.key, self.n_ref, self.order = key, n_ref, order
        bf = torch.bfloat16
        self.h1 = torch.empty(B, N, d, device=device, dtype=bf)
        self.r_ref = torch.zeros(B, N, d, device=device, dtype=bf)
        self.r_new = torch.empty(B, N, d, device=device, dtype=bf)
        self.h1c = torch.empty(B, n_seq, d, device=device, dtype=bf)
        self.R = self.R_slots = self.ctl = None
        if order == 0:
            self.R = torch.empty(B, n_seq, d, device=device, dtype=torch.float32)
        else:
            self.R_slots = torch.zeros(order + 1, B, n_seq, d, device=device, dtype=torch.float32)
            self.slot_sigma = [None] * (order + 1)
            self.n_computed = 0
            # slot -1 and zero coefficients until the first write: an update writes nothing and an apply reads nothing
            self.ctl = torch.tensor([-1, 0, 0, 0], device=device, dtype=torch.int32)
            self.ctl_slot, self.ctl_coef = self.ctl[:1], self.ctl[1:].view(torch.float32)
            cuda = torch.device(device).type == "cuda"
            self._staging = torch.empty(4, dtype=torch.int32, pin_memory=cuda)
            self._staged = torch.cuda.Event() if cuda else None
        self.partials = torch.empty(ops.STEP_CACHE_PARTIALS, device=device, dtype=torch.float32)
        self.out = torch.zeros(4, device=device, dtype=torch.float64)

    def indicator(self, h0):
        """Launch the indicator of h0 (the patch embedding) and self.h1 (block 0's output)."""
        return ops.step_cache_indicator(h0, self.h1, self.r_ref, self.r_new, self.h1c, self.n_ref, self.partials, self.out)

    def read_indicator(self):
        """The host's one 16-byte device-to-host copy per step: the two sums -> the indicator.  The copy is blocking, so the
        host waits here for everything enqueued on the stream before it (write_control relies on this)."""
        num, den = self.out[:2].tolist()
        return indicator(num, den)

    def write_control(self, slot, coef):
        """One stream-ordered host-to-device copy of (slot, coef[0..2]) into the control block, for the tail that follows.
        The copy reads the pinned staging buffer when it executes, so the staging buffer must not be rewritten before then.
        Every step reads its indicator (read_indicator, a blocking copy on the same stream) before it writes its control,
        so the previous step's copy has executed by now; the event wait states that dependency and returns at once."""
        if self._staged is not None:
            self._staged.synchronize()
        st = self._staging.numpy()
        st[0] = slot
        st[1:] = np.asarray(coef, dtype=np.float32).view(np.int32)
        self.ctl.copy_(self._staging, non_blocking=True)
        if self._staged is not None:
            self._staged.record()

    def nbytes(self):
        R = self.R if self.R is not None else self.R_slots
        return sum(t.numel() * t.element_size() for t in (self.h1, self.r_ref, self.r_new, self.h1c, R))


class FirstBlockCache:
    """State of one sampling run.  `threshold` (float >= 0, inf allowed) may be changed between steps.  `history` lists
    (indicator, skipped) for every forward since the last reset().

    order (0, 1 or 2): the degree of the forecast of the skipped blocks' residual.  0 holds R of the last computed step;
    1 and 2 extrapolate it in the sampler's sigma from the last 2 or 3 computed steps (see the module docstring), at the
    cost of order + 1 fp32 slots of [B, n_seq, d] instead of one (+0.88 GB per order at 512x512, +1.54 GB at 512x896,
    b = 2).  At order >= 1 every forward needs the sigma of its step: sampler_step and GraphedStep pass it (set_sigma).
    max_skips (None or an int >= 0): after that many consecutive skipped steps the next one computes whatever its indicator
    says (0: never skip).  No default order or max_skips is chosen, as for the threshold."""

    def __init__(self, threshold, order=0, max_skips=None):
        self.threshold = threshold
        self._order = check_order(order)
        self.max_skips = max_skips
        self._sigma = None
        self.reset()

    @property
    def threshold(self):
        return self._threshold

    @threshold.setter
    def threshold(self, value):
        self._threshold = check_threshold(value)

    @property
    def order(self):
        return self._order

    @property
    def max_skips(self):
        return self._max_skips

    @max_skips.setter
    def max_skips(self, value):
        self._max_skips = check_max_skips(value)

    def reset(self):
        """Drop all state and buffers (the forecast slots and their sigmas with them): the next forward computes."""
        self.buffers = None
        self.has_state = False
        self.history = []
        self._run = 0  # consecutive skipped steps
        self._step_sigma = None

    def set_sigma(self, sigma):
        """The sampler's sigma of the next forward (a host value).  The forward consumes it; order >= 1 requires it."""
        self._sigma = check_sigma(sigma)

    def begin(self):
        """Start a forward: consume the sigma given by set_sigma.  Raises ValueError at order >= 1 when there is none, before
        anything is launched."""
        sigma, self._sigma = self._sigma, None
        if self._order >= 1 and sigma is None:
            raise ValueError(f"step_cache: a FirstBlockCache of order {self._order} needs the sampler's sigma of every step "
                             "before the forward (step_cache.set_sigma(sigma)); sampler_step and GraphedStep pass it")
        self._step_sigma = sigma

    def workspace(self, B, N, d, n_ref, n_seq, device):
        """The buffers of this geometry; a different key than the current one drops the state and the old buffers."""
        key = (int(B), int(N), int(d), int(n_ref), int(n_seq), torch.device(device))
        if self.buffers is None or self.buffers.key != key:
            self.buffers, self.has_state = None, False  # free the old set before allocating the new one
            self.buffers = Buffers(key, self._order)
        return self.buffers

    def decide(self, ind):
        """Skip iff there is state for the current buffers, ind < threshold and fewer than max_skips steps in a row were
        skipped.  Records (ind, skipped) in history."""
        skip = bool(self.has_state and ind < self._threshold and (self._max_skips is None or self._run < self._max_skips))
        self._run = self._run + 1 if skip else 0
        self.history.append((ind, skip))
        return skip

    def control(self, skip):
        """(slot, coefficients) of this step at order >= 1: a computed step writes slot n_computed mod (order + 1) and applies
        nothing; a skipped step writes no slot (-1) and applies the forecast at this step's sigma."""
        b = self.buffers
        if not skip:
            return b.n_computed % (self._order + 1), [0.0] * (self._order + 1)
        return -1, forecast_coefficients(self._step_sigma, b.slot_sigma, b.n_computed, self._order)

    def stage(self, skip):
        """After decide(): at order >= 1, write this step's control block for the tail (nothing at order 0)."""
        if self._order >= 1:
            slot, coef = self.control(skip)
            self.buffers.write_control(slot, coef + [0.0] * (3 - len(coef)))

    def computed(self):
        """After a computed step: R (or, at order >= 1, the slot control() named, now tagged with this step's sigma) holds its
        residual and r_new its r, which becomes r_ref (swap, no copy)."""
        b = self.buffers
        b.r_ref, b.r_new = b.r_new, b.r_ref
        if self._order >= 1:
            b.slot_sigma[b.n_computed % (self._order + 1)] = self._step_sigma
            b.n_computed += 1
        self.has_state = True
