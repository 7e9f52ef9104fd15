"""CFG-Zero* guidance (Fan et al., 2025, "CFG-Zero*: Improved Classifier-Free Guidance for Flow Matching Models"): an
opt-in replacement for the sampler's vanilla guidance g = u + s (c - u).

This module is the only one that knows the rule.  It makes two changes:

  optimised scale   the unconditional output is scaled by s* = <c, u> / (|u|^2 + 1e-8), one scalar over all latent
                    elements of the sample, before the usual combine: g = s* u + s (c - s* u).  When u is all zero s* = 0
                    and g = s c; a NaN propagates.
  zero-init         the first k sampler steps since reset() use a velocity of exactly zero, so no model output is needed
                    and their forward is skipped: with Euler x stays as it is; a UniPC solver steps on a zero CFG pair,
                    so its history holds m = x - sigma * 0 = x and stays in step with its schedule.  The paper's code
                    zeroes step 0 only, which is k = 1.

On the device (ops.cfg_zero_scale, then a scaled update): pass 1 adds f32(c) u and u u per CTA in fp32 over a partition
fixed by the size; pass 2 adds the CTA sums in fp64 in a fixed order and writes s* = dot / (norm + 1e-8), computed in fp64
and rounded once to fp32, to a one-float device buffer that the update kernels read through a pointer.  s* never goes to
the host, so no step adds a host synchronisation and no captured graph depends on it.  u is formed as the update forms
it: from the CFG pair on a full step, and as f32(c) - delta (or its forecast) on a CFG cache's conditional-only step.
Each update then forms u' = s* u (one rounded product) and runs its usual instructions on u' in place of u.

Memory per (latent shape, device): the reduction's fp32 partials (8 KiB), an fp64 {dot, norm, 0, 0} and one fp32 s*;
with a UniPC solver and k >= 1, also a zero bf16 CFG pair (4 bytes per latent element).  No default k is chosen: what
real weights want is not measured here.
"""
import numbers

import torch

from . import ops


def check_guidance(guidance):
    """None or a CFGZeroStar; anything else is a TypeError naming guidance."""
    if guidance is not None and not isinstance(guidance, CFGZeroStar):
        raise TypeError(f"guidance must be a scail_b200.guidance.CFGZeroStar or None, got {type(guidance).__name__}")
    return guidance


def check_supported(cp=None, chunk_dim=None):
    """Refuse what the rule does not cover: under context parallelism (size > 1) or with chunk_dim a rank may hold only part
    of the velocity, so its s* would be a partial sum."""
    if cp is not None and getattr(cp, "size", 1) > 1:
        raise NotImplementedError(f"guidance is not implemented under context parallelism (a ContextParallel of size "
                                  f"{cp.size}): s* would be a partial sum; run without guidance or on one GPU")
    if chunk_dim is not None:
        raise NotImplementedError("guidance is not implemented with chunk_dim (pre-chunked sequence parallelism): s* would "
                                  "be a partial sum")


class _Buffers:
    """The device state for one latent (shape, device): the reduction's partials, its fp64 result {dot, norm, 0, 0}, the
    fp32 s* the updates read, and (on first use) a zero bf16 CFG pair for the solver's zero-initialised steps."""

    def __init__(self, key):
        shape, device = key
        self.key = key
        self.partials = torch.empty(ops.STEP_CACHE_PARTIALS, device=device, dtype=torch.float32)
        self.out = torch.zeros(4, device=device, dtype=torch.float64)
        self.u_scale = torch.zeros(1, device=device, dtype=torch.float32)
        self.zero_pair = None


class CFGZeroStar:
    """CFG-Zero* state of one sampling run, for sampler.sample / sampler_step / GraphedStep / sample_long(guidance=).

    zero_init_steps (an int >= 0): steps 0 .. k-1 since reset() are zero-initialised, every later step is guided with s*;
    0 keeps only the optimised scale.  sample() and GraphedStep() call reset()."""

    def __init__(self, zero_init_steps=1):
        if isinstance(zero_init_steps, bool) or not isinstance(zero_init_steps, numbers.Integral) or zero_init_steps < 0:
            raise ValueError(f"CFGZeroStar: zero_init_steps must be an int >= 0, got {zero_init_steps!r}")
        self._k = int(zero_init_steps)
        self._bufs = {}
        self.reset()

    @property
    def zero_init_steps(self):
        return self._k

    def reset(self):
        """The next step is step 0 again.  Buffers are kept: every step writes s* before an update reads it."""
        self._i = 0
        self._last = None

    @property
    def step_index(self):
        """Steps counted since reset()."""
        return self._i

    def begin_step(self):
        """Count one sampler step; True iff it is zero-initialised (one of the first zero_init_steps since reset())."""
        zero = self._i < self._k
        self._i += 1
        return zero

    @property
    def last_scale(self):
        """The fp32 [1] device tensor holding the last s* written (None before the first), for tests; it is overwritten by
        the next reduction on a latent of the same shape and device."""
        return self._last

    def _buffers(self, shape, device):
        key = (tuple(shape), torch.device(device))
        b = self._bufs.get(key)
        if b is None:
            b = self._bufs[key] = _Buffers(key)
        return b

    def scale(self, v, delta=None, forecast=None):
        """Launch the reduction (ops.cfg_zero_scale) on the current stream and return s* as an fp32 [1] device tensor: from
        the CFG pair v (bf16 [2, ...]), or from c = v (bf16 [1, ...]) and u = f32(c) - delta, or f32(c) - the forecast
        (slots, coefficients) of a CFG cache of order >= 1."""
        b = self._buffers((1, *v.shape[1:]), v.device)
        ops.cfg_zero_scale(v, b.partials, b.out, b.u_scale, delta=delta, forecast=forecast)
        self._last = b.u_scale
        return b.u_scale

    def zero_pair(self, x):
        """A zero bf16 CFG pair [2, *x.shape[1:]] on x's device: the solver's input on a zero-initialised step."""
        b = self._buffers((1, *x.shape[1:]), x.device)
        if b.zero_pair is None:
            b.zero_pair = torch.zeros((2, *x.shape[1:]), device=x.device, dtype=torch.bfloat16)
        return b.zero_pair

    def zero_step(self, x, scale, sigma, next_sigma, solver=None):
        """A zero-initialised step in place on x: nothing with Euler; solver.step on a zero pair with a UniPC.  Returns x."""
        if solver is not None:
            solver.step(x, self.zero_pair(x), scale, sigma, next_sigma)
        return x

    def update(self, x, v, scale, sigma, next_sigma, solver=None):
        """A guided full step in place on x from the CFG pair v: s* from v, then the scaled Euler step or solver.step."""
        s = self.scale(v)
        if solver is not None:
            return solver.step(x, v, scale, sigma, next_sigma, u_scale=s)
        return ops.cfg_euler_(x, v, scale, float(next_sigma) - float(sigma), u_scale=s)
