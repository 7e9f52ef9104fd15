"""Opt-in replacements for the sampler's vanilla guidance g = u + s (c - u): CFG-Zero* and APG.  This module is the only one
that knows their rules.

CFG-Zero* (Fan et al., 2025, "CFG-Zero*: Improved Classifier-Free Guidance for Flow Matching Models") makes two changes:

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

APG, adaptive projected guidance (Sadat, Hilliges, Weber, "Eliminating Oversaturation and Artifacts of High Guidance
Scales in Diffusion Models", ICLR 2025), guides in data-prediction space.  For a step from sigma to sigma' with guidance
scale w (the sampler's scale), on the latent x [1, T, 16, h, w]:

  D_c = x - sigma c,  D_u = x - sigma u,  diff = D_c - D_u
  momentum beta       avg <- diff + beta avg;  diff <- avg            (avg: one fp32 latent, zero after reset(); 0 = off)
  norm threshold r    per frame t: diff_t <- diff_t min(1, r / |diff_t|)   (0 = off; factor 1 when |diff_t| = 0)
  projection          per frame t: par_t = (<diff_t, D_c,t> / |D_c,t|^2) D_c,t (0 when |D_c,t| = 0), orth_t = diff_t - par_t
  D_g = D_c + (w - 1) (orth + eta par)
  Euler: x' = x + (sigma' - sigma) (x - D_g) / sigma;   UniPC: D_g is the step's data prediction m.

A frame is one latent frame x[0, t], 16 h w contiguous elements: the paper's per-image rule applied to each frame of the
video.  With eta = 1, beta = 0 and r = 0 the step is vanilla CFG in exact arithmetic.  NaN propagates.

On the device (ops.apg_reduce, ops.apg_finish, then ops.apg_update_): pass 1 forms D_c and diff per element, applies the
momentum (reading and writing avg once: this pass owns the write, and the update reads the new avg as diff) and adds
diff*diff, diff*D_c and D_c*D_c per (frame, CTA) in fp32 over a partition fixed by the shape; pass 2 adds each frame's
partials in fp64 in a fixed order and writes the threshold factor f_t and the projection coefficient p_t = f_t <diff_t,
D_c,t> / |D_c,t|^2, each rounded once to fp32, to a [T, 2] device buffer; the update applies the rule, then the Euler step
in place or D_g into an fp32 buffer that the solver's data-prediction step reads.  The factors never go to the host, so no
step adds a host synchronisation and no captured graph depends on them.  u is formed as the update forms it: from the CFG
pair on a full step, as f32(c) - delta (or its forecast) on a CFG cache's conditional-only step, and the momentum advances
on every guided step, full or conditional-only.

Memory per (latent shape, device): with momentum one fp32 latent (16.5 MB at 512x512 and 28.9 MB at 512x896, as every
latent copy here); with a UniPC solver one fp32 latent for D_g; 3 T 32 fp32 partials, T x 4 fp64 sums and T x 2 fp32
factors.  APG is not available in sample_long (momentum would need state per window) or guided_velocity.  No default
eta, r or beta is chosen: what real weights want is not measured here.
"""
import math
import numbers

import torch

from . import ops


def check_guidance(guidance):
    """None, a CFGZeroStar or an APG; anything else is a TypeError naming guidance."""
    if guidance is not None and not isinstance(guidance, (CFGZeroStar, APG)):
        raise TypeError("guidance must be a scail_b200.guidance.CFGZeroStar, a scail_b200.guidance.APG or None, got "
                        f"{type(guidance).__name__}")
    return guidance


def check_supported(cp=None, chunk_dim=None):
    """Refuse what the rules do not cover: under context parallelism (size > 1) or with chunk_dim a rank may hold only part
    of the velocity, so CFG-Zero*'s s* and APG's per-frame sums would be partial sums."""
    if cp is not None and getattr(cp, "size", 1) > 1:
        raise NotImplementedError(f"guidance is not implemented under context parallelism (a ContextParallel of size "
                                  f"{cp.size}): s* or APG's per-frame sums would be partial sums; run without guidance or "
                                  "on one GPU")
    if chunk_dim is not None:
        raise NotImplementedError("guidance is not implemented with chunk_dim (pre-chunked sequence parallelism): s* or "
                                  "APG's per-frame sums would be partial sums")


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


def _check_real(name, value, nonneg=False):
    """A finite real number (not a bool) -> float; else ValueError naming the argument."""
    ok = isinstance(value, numbers.Real) and not isinstance(value, bool) and math.isfinite(value)
    if not ok or (nonneg and value < 0):
        raise ValueError(f"APG: {name} must be a finite {'real >= 0' if nonneg else 'real'}, got {value!r}")
    return float(value)


class _APGBuffers:
    """The device state for one latent (shape, device): pass 1's partials, pass 2's fp64 sums [T, 4] and fp32 factors [T, 2],
    the momentum average (fp32, the latent's shape; with momentum only) and, on first use with a solver, D_g."""

    def __init__(self, key, momentum):
        shape, device = key
        T = shape[1]
        self.key = key
        self.partials = torch.empty(ops.apg_partials_len(T), device=device, dtype=torch.float32)
        self.sums = torch.zeros(T, 4, device=device, dtype=torch.float64)
        self.factors = torch.zeros(T, 2, device=device, dtype=torch.float32)
        self.avg = torch.zeros(shape, device=device, dtype=torch.float32) if momentum else None
        self.stale = False  # the average holds a run before reset(): zero it before the next read
        self.m = None


class APG:
    """APG state of one sampling run, for sampler.sample / sampler_step / GraphedStep(guidance=); see the module docstring.

    eta (finite real): the weight of the component of diff parallel to D_c; eta = 1 with r = 0 and momentum = 0 is vanilla
    CFG.  norm_threshold r (finite real >= 0; 0 = off): each frame's diff is scaled down to norm r, in data-prediction units
    per frame, so its meaning depends on the frame's size 16 h w: the same r bounds the per-element difference more tightly
    on a larger latent.  momentum beta (finite real; 0 = off, the paper uses beta < 0): avg <- diff + beta avg, over the
    guided steps since reset().  Bools, non-finite values and a negative r raise ValueError naming the argument.  sample()
    and GraphedStep() call reset()."""

    def __init__(self, eta, norm_threshold=0.0, momentum=0.0):
        self._eta = _check_real("eta", eta)
        self._r = _check_real("norm_threshold", norm_threshold, nonneg=True)
        self._beta = _check_real("momentum", momentum)
        self._bufs = {}
        self.reset()

    @property
    def eta(self):
        return self._eta

    @property
    def norm_threshold(self):
        return self._r

    @property
    def momentum(self):
        return self._beta

    def reset(self):
        """Zero the momentum average (before its next read) and the step count.  The other buffers are kept: every step
        writes them before it reads them."""
        self._i = 0
        self._last = None
        for b in self._bufs.values():
            b.stale = True

    @property
    def step_index(self):
        """Guided steps counted since reset()."""
        return self._i

    def begin_step(self):
        """Count one sampler step; always False: APG has no zero-initialised step (the sampler's CFG-Zero* hook)."""
        self._i += 1
        return False

    @property
    def last_factors(self):
        """The fp32 [T, 2] device tensor of the last per-frame (threshold factor, projection coefficient), None before the
        first, for tests; it is overwritten by the next step on a latent of the same shape and device."""
        return self._last

    def _buffers(self, x):
        key = (tuple(x.shape), torch.device(x.device))
        b = self._bufs.get(key)
        if b is None:
            b = self._bufs[key] = _APGBuffers(key, self._beta != 0.0)
        if b.stale:
            if b.avg is not None:
                b.avg.zero_()
            b.stale = False
        return b

    def update(self, x, v, scale, sigma, next_sigma, solver=None, delta=None, forecast=None):
        """A guided step in place on x (fp32 [1, T, 16, h, w]) at sigma > 0: the two reductions, then the Euler step, or D_g
        into this object's buffer and solver.step(m=D_g) with a UniPC.  u and c come from the CFG pair v, or from c = v
        alone with delta or forecast (a CFGCache's conditional-only step), as ops.apg_reduce takes them.  Returns x."""
        sigma = float(sigma)
        if not sigma > 0.0:
            raise ValueError(f"APG: a guided step needs sigma > 0 (data predictions divide by it), got {sigma!r}")
        if solver is not None:
            solver.check_step(x, sigma, next_sigma)
        b = self._buffers(x)
        ops.apg_reduce(x, v, sigma, b.partials, b.avg, self._beta, delta=delta, forecast=forecast)
        ops.apg_finish(b.partials, b.sums, b.factors, self._r, x.shape[1], x.numel())
        self._last = b.factors
        if solver is None:
            return ops.apg_update_(x, v, b.factors, scale, self._eta, sigma, next_sigma, avg=b.avg, delta=delta,
                                   forecast=forecast)
        if b.m is None:
            b.m = torch.empty_like(x)
        ops.apg_update_(x, v, b.factors, scale, self._eta, sigma, out=b.m, avg=b.avg, delta=delta, forecast=forecast)
        return solver.step(x, None, scale, sigma, next_sigma, m=b.m)
