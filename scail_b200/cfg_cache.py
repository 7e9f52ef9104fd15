"""CFG cache: run only the conditional branch of the DiT on sampler steps where the CFG difference has settled.

Every sampler step runs the DiT on the CFG batch [uncond, cond] (b = 2).  The difference delta = c - u of the two outputs
changes slowly over late steps, so some steps can run the conditional branch alone (b = 1) and rebuild the unconditional
output as u = c - delta, with delta from the last full step (order 0, a hold) or forecast in sigma from the last full
steps (order >= 1, below).  This module owns the policy:

  full step         the b = 2 forward, then ops.cfg_cache_delta: delta_new = f32(c) - f32(u) (fp32 [1, t, 16, h, w], one
                    subtraction rounded once) and the sums num = sum|delta_new - delta_ref|, den = sum|delta_ref|, where
                    delta_ref is delta of the previous full step (zero-filled at allocation, so the first full step's
                    indicator num / den is +inf); then delta_ref <- delta_new (a buffer swap).  The latent update is the
                    usual cfg_euler_ / UniPC.step on the pair.
  decision          on the host before each step's forward: conditional-only iff the cache holds a delta, the indicator of
                    the last full step is < threshold (a NaN never skips) and fewer than max_skips steps in a row were
                    conditional-only.  The sums are read with one blocking 16-byte device-to-host copy, when the next step
                    decides.  So threshold 0 never skips, at threshold inf steps 0 and 1 are full and every later step is
                    conditional-only, and max_skips=1 at inf alternates.
  conditional-only  the b = 1 forward on the cond row (timesteps [1], context[1:2], the other inputs unchanged), on a
                    stream the cache owns (CFGCache.stream), joined to the caller's stream both ways; then the fused
                    update with u = f32(c) - delta_ref: ops.cfg_euler_cached_ or UniPC.step(delta=).

The cache's stream exists because the DiT's workspace is kept per stream and reallocated when its shapes change: b = 1
and b = 2 forwards alternating on one stream would reallocate it on every switch.  The stream holds one b = 1 workspace,
which is dropped when the cache is garbage-collected.  torch.cuda.Stream() hands out stream handles from a pool, so two
objects may still come to share one handle and hence one workspace; for eager forwards that costs a reallocation at most,
and GraphedStep keeps the workspace tensors its graphs were captured against (see sampler.GraphedStep), so no graph ever
reads freed memory.  No default threshold is chosen: that needs real weights and a visual check.

Taylor forecast (order >= 1).  Instead of holding delta, the cache keeps delta of the last order + 1 full steps, each with
the sampler's sigma of its step, in order + 1 fp32 slots shaped like the latent (zero-filled at allocation); the j-th full
step since reset() writes slot j mod (order + 1).  The forecast at sigma is step_cache.forecast_coefficients(sigma, slot
sigmas, full steps so far, order): the Lagrange polynomial in sigma through the m + 1 most recent full steps, m = min(order,
full steps - 1), reduced until their sigmas are pairwise distinct, with its fp64 coefficients rounded once to fp32 (the
first-block cache's forecast).  On the device delta_hat = c0*S0, then + c1*S1, then + c2*S2, every product and sum rounded
on its own, and a slot whose coefficient is 0 is not read.

  full step j       ops.cfg_cache_delta_forecast: slot j mod (order + 1) = f32(c) - f32(u), and the sums num = sum|delta_j -
                    delta_hat|, den = sum|delta_hat| against the forecast at sigma_j from the j earlier full steps, so the
                    indicator measures how far the forecast was off.  At j = 0 every coefficient is 0 (+inf); at j = 1 the
                    forecast is the hold, and the sums are cfg_cache_delta's bit for bit.  The slot written may be the oldest
                    one the forecast reads: the kernel reads all of an element before it writes it.
  decision          unchanged.
  conditional-only  u = f32(c) - delta_hat(sigma) from the order + 1 most recent full steps: ops.cfg_euler_cached_forecast_
                    or UniPC.step(forecast=).

The coefficients are kernel arguments, so nothing here is captured in a graph.  Each step needs its sigma on the host
(begin_step(x, sigma)); sampler_step and GraphedStep pass it.  Memory: order + 1 fp32 latents instead of 2 (16.5 MB at
512x512 and 29 MB at 512x896 at order 2).  No default order is chosen either.
"""
import weakref

import torch

from . import ops
from .guidance import APG
from .step_cache import check_max_skips, check_order, check_sigma, check_threshold, forecast_coefficients, indicator

def _drop_workspaces(handles):
    """Free the per-stream DiT workspace of the given stream handles (a CFGCache's streams, once it is collected)."""
    from . import dit
    for key in [k for k in dit._WS.bufs if k[0][1] in handles]:
        del dit._WS.bufs[key]


def check_supported(cp=None, chunk_dim=None, num_layers=None, plan=None):
    """Refuse what the cache does not cover: under context parallelism or a hybrid CFG plan every rank would have to agree on
    the decision (and a HybridParallel uncond rank would idle on conditional-only steps), and a truncated or pre-chunked
    forward is not a full step."""
    if cp is not None and getattr(cp, "size", 1) > 1:
        raise NotImplementedError(f"cfg_cache is not implemented under context parallelism (a ContextParallel of size {cp.size}); "
                                  "run without a CFG cache or on one GPU")
    if plan is not None:
        raise NotImplementedError("cfg_cache is not implemented with a HybridParallel plan: its uncond rank would idle on "
                                  "conditional-only steps; run without a CFG cache or on one GPU")
    if chunk_dim is not None:
        raise NotImplementedError("cfg_cache is not implemented with chunk_dim (pre-chunked sequence parallelism)")
    if num_layers is not None:
        raise NotImplementedError("cfg_cache is not implemented with _num_layers: a truncated forward is not a sampler step")


def check_cache(cfg_cache):
    """None or a CFGCache; anything else is a TypeError naming cfg_cache."""
    if cfg_cache is not None and not isinstance(cfg_cache, CFGCache):
        raise TypeError(f"cfg_cache must be a scail_b200.cfg_cache.CFGCache or None, got {type(cfg_cache).__name__}")
    return cfg_cache


class Buffers:
    """The cache's device state for one latent (shape, device): delta_ref and delta_new (fp32, the latent's shape; delta_ref
    zero-filled), the delta kernel's partial sums and its fp64 result {num, den, ratio, 0}.  At order >= 1, d_ref and d_new
    are None and `slots` (fp32 [order + 1, *shape], zero-filled) takes their place, with slot_sigma (the sigma of the full
    step each slot holds, None while empty) and n_full (full steps written since allocation)."""

    def __init__(self, key, order=0):
        shape, device = key
        self.key = key
        self.d_ref = self.d_new = self.slots = None
        if order == 0:
            self.d_ref = torch.zeros(shape, device=device, dtype=torch.float32)
            self.d_new = torch.empty(shape, device=device, dtype=torch.float32)
        else:
            self.slots = torch.zeros((order + 1, *shape), device=device, dtype=torch.float32)
            self.slot_sigma = [None] * (order + 1)
            self.n_full = 0
        self.partials = torch.empty(ops.STEP_CACHE_PARTIALS, device=device, dtype=torch.float32)
        self.out = torch.zeros(4, device=device, dtype=torch.float64)

    def read_indicator(self):
        """The host's one 16-byte device-to-host copy: the two sums -> the indicator (blocking)."""
        num, den = self.out[:2].tolist()
        return indicator(num, den)

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.d_ref, self.d_new, self.slots) if t is not None)


class CFGCache:
    """State of one sampling run, for sampler.sample / sampler_step / GraphedStep(cfg_cache=).

    threshold (float >= 0, inf allowed; validated as FirstBlockCache's) may change between steps.  max_skips (None or an
    int >= 0): after that many conditional-only steps in a row the next step is full (0: never skip).  `history` lists
    (indicator, cond_only) for every step since reset(): the indicator the step decided on, i.e. that of the last full
    step, or None while the cache holds no delta.

    order (0, 1 or 2; validated as FirstBlockCache's): the degree of the forecast of delta in the sampler's sigma.  0 holds
    delta of the last full step; 1 and 2 extrapolate it from the last 2 or 3 full steps and measure each full step against
    that forecast (see the module docstring), at the cost of order + 1 fp32 latents instead of 2.  At order >= 1 every
    step needs its sigma (begin_step(x, sigma)); sampler_step and GraphedStep pass it."""

    def __init__(self, threshold, max_skips=None, order=0):
        self.threshold = threshold
        self.max_skips = max_skips
        self._order = check_order(order, "cfg_cache")
        self._streams = {}  # device index -> this cache's stream for the conditional-only forward
        self._handles = set()  # every stream handle this cache ran a forward on: their workspaces go with the cache
        weakref.finalize(self, _drop_workspaces, self._handles)
        self.reset()

    @property
    def threshold(self):
        return self._threshold

    @threshold.setter
    def threshold(self, value):
        self._threshold = check_threshold(value, "cfg_cache")

    @property
    def order(self):
        return self._order

    @property
    def max_skips(self):
        return self._max_skips

    @max_skips.setter
    def max_skips(self, value):
        self._max_skips = check_max_skips(value, "cfg_cache")

    def reset(self):
        """Drop the held delta and its buffers (the forecast slots and their sigmas with them): the next two steps are full."""
        self.buffers = None
        self._ind = None  # indicator of the last full step; None while no delta is held
        self._pending = False  # the last full step's sums are on the device, not yet read
        self._run = 0  # consecutive conditional-only steps
        self._sigma = None  # sigma of the current step (order >= 1)
        self.history = []

    @property
    def delta(self):
        """c - u of the last full step (fp32, the latent's shape: delta_ref, or at order >= 1 its slot), or None."""
        b = self.buffers
        if b is None or self._order == 0:
            return None if b is None else b.d_ref
        return None if b.n_full == 0 else b.slots[(b.n_full - 1) % (self._order + 1)]

    def decide(self, ind):
        """The pure rule: ind is the indicator of the last full step, or None when no delta is held.  Conditional-only iff
        ind is not None, ind < threshold (never for NaN) and fewer than max_skips steps in a row were conditional-only.
        Records (ind, cond_only) in history."""
        cond_only = bool(ind is not None and ind < self._threshold and (self._max_skips is None or self._run < self._max_skips))
        self._run = self._run + 1 if cond_only else 0
        self.history.append((ind, cond_only))
        return cond_only

    def begin_step(self, x, sigma=None):
        """Before a step's forward on the latent x at the sampler's `sigma`: read the last full step's sums if they are still
        on the device, then decide.  A latent of another shape or device than the held delta's drops the state first.  At
        order >= 1 sigma is required: without it, ValueError before anything is read or recorded."""
        if self._order >= 1:
            if sigma is None:
                raise ValueError(f"cfg_cache: a CFGCache of order {self._order} needs the sampler's sigma of every step "
                                 "(begin_step(x, sigma)); sampler_step and GraphedStep pass it")
            self._sigma = check_sigma(sigma, "cfg_cache")
        if self.buffers is not None and self.buffers.key != (tuple(x.shape), x.device):
            self.buffers, self._ind, self._pending = None, None, False
        if self._pending:
            self._ind = self.buffers.read_indicator()
            self._pending = False
        return self.decide(self._ind)

    def full_control(self):
        """(slot, coefficients) of the next full step at order >= 1: it writes slot n_full mod (order + 1) and measures
        against the forecast at this step's sigma from the earlier full steps (all zero before the first)."""
        b = self.buffers
        return b.n_full % (self._order + 1), forecast_coefficients(self._sigma, b.slot_sigma, b.n_full, self._order)

    def forecast(self):
        """The coefficients of delta_hat at this step's sigma from the order + 1 most recent full steps (order >= 1)."""
        b = self.buffers
        return forecast_coefficients(self._sigma, b.slot_sigma, b.n_full, self._order)

    def full_step(self, v):
        """After a full step's forward, v the bf16 CFG pair [2, t, 16, h, w]: launch the delta kernel and swap delta_ref and
        delta_new (at order >= 1: write the next slot, tag it with this step's sigma).  The sums are read by the next
        begin_step."""
        key = ((1, *v.shape[1:]), v.device)
        if self.buffers is None:
            self.buffers = Buffers(key, self._order)
        b = self.buffers
        if self._order == 0:
            ops.cfg_cache_delta(v, b.d_ref, b.d_new, b.partials, b.out)
            b.d_ref, b.d_new = b.d_new, b.d_ref
        else:
            slot, coef = self.full_control()
            ops.cfg_cache_delta_forecast(v, b.slots, slot, coef, b.partials, b.out)
            b.slot_sigma[slot] = self._sigma
            b.n_full += 1
        self._pending = True

    def cond_update(self, x, c, scale, sigma, next_sigma, solver=None, guidance=None):
        """The conditional-only step's latent update in place on x from c, the conditional output alone (bf16 [1, ...]): u =
        f32(c) - delta (order 0) or f32(c) - delta_hat(sigma) (order >= 1), then the Euler step, or solver.step (a UniPC)
        when given.  With guidance (a scail_b200.guidance.CFGZeroStar), s* is reduced from that same u first and the
        update is the scaled one; with a scail_b200.guidance.APG, its step runs on that same u.  Returns x."""
        if isinstance(guidance, APG):
            kw = dict(delta=self.delta) if self._order == 0 else dict(forecast=(self.buffers.slots, self.forecast()))
            return guidance.update(x, c, scale, sigma, next_sigma, solver, **kw)
        ds = float(next_sigma) - float(sigma)
        if self._order == 0:
            kw = {} if guidance is None else dict(u_scale=guidance.scale(c, delta=self.delta))
            if solver is not None:
                return solver.step(x, c, scale, sigma, next_sigma, delta=self.delta, **kw)
            return ops.cfg_euler_cached_(x, c, self.delta, scale, ds, **kw)
        fc = (self.buffers.slots, self.forecast())
        kw = {} if guidance is None else dict(u_scale=guidance.scale(c, forecast=fc))
        if solver is not None:
            return solver.step(x, c, scale, sigma, next_sigma, forecast=fc, **kw)
        return ops.cfg_euler_cached_forecast_(x, c, *fc, scale, ds, **kw)

    def stream(self, device):
        """This cache's stream for the conditional-only forward on `device`, created on first use.  Should the caller come
        to run on that very stream, the cache draws another one: the b = 1 and b = 2 workspaces must not share a stream."""
        dev = torch.device(device)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        s = self._streams.get(idx)
        if s is None or s.cuda_stream == torch.cuda.current_stream(idx).cuda_stream:
            s = self._streams[idx] = torch.cuda.Stream(device=idx)
        return s

    def cond_forward(self, model, x, timesteps, context, kw):
        """The conditional-only forward, model(x, timesteps=timesteps, context=context, **kw) with x [1, ...] and context
        the cond row, on stream() after everything enqueued on the current stream; the current stream then waits for it.
        With fp8_linear the 8-bit weights of its mode are brought up to date on the current stream first.  -> v bf16 [1, ...]."""
        dev = x.device
        main = torch.cuda.current_stream(dev)
        side = self.stream(dev)
        self._handles.add(side.cuda_stream)
        ad = model.mixins["adaln_layer"] if hasattr(model, "mixins") else None
        if ad is not None and getattr(ad, "fp8_linear", False):
            ad.prepare_fp8_weights(streams=(side,))
        side.wait_stream(main)
        with torch.cuda.stream(side):
            v = model(x, timesteps=timesteps, context=context, **kw).contiguous()
        main.wait_stream(side)
        v.record_stream(main)
        return v
