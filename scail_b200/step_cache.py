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
"""
import math
import numbers

import torch

from . import ops


def check_threshold(threshold):
    """A float >= 0 (inf allowed).  Raises TypeError for bools and non-numbers, ValueError for NaN and negatives."""
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real):
        raise TypeError(f"step cache threshold must be a real number >= 0 (inf allowed), got {threshold!r}")
    t = float(threshold)
    if math.isnan(t) or t < 0:
        raise ValueError(f"step cache threshold must be >= 0 (inf allowed), got {threshold!r}")
    return t


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
    h1, bf16) and R (fp32 [B, n_seq, d]), plus the indicator's partial sums and its fp64 result {num, den, ratio, 0}."""

    def __init__(self, key):
        B, N, d, n_ref, n_seq, device = key
        self.key, self.n_ref = key, n_ref
        bf = torch.bfloat16
        self.h1 = torch.empty(B, N, d, device=device, dtype=bf)
        self.r_ref = torch.zeros(B, N, d, device=device, dtype=bf)
        self.r_new = torch.empty(B, N, d, device=device, dtype=bf)
        self.h1c = torch.empty(B, n_seq, d, device=device, dtype=bf)
        self.R = torch.empty(B, n_seq, d, device=device, dtype=torch.float32)
        self.partials = torch.empty(ops.STEP_CACHE_PARTIALS, device=device, dtype=torch.float32)
        self.out = torch.zeros(4, device=device, dtype=torch.float64)

    def indicator(self, h0):
        """Launch the indicator of h0 (the patch embedding) and self.h1 (block 0's output)."""
        return ops.step_cache_indicator(h0, self.h1, self.r_ref, self.r_new, self.h1c, self.n_ref, self.partials, self.out)

    def read_indicator(self):
        """The host's one 16-byte device-to-host copy per step: the two sums -> the indicator."""
        num, den = self.out[:2].tolist()
        return indicator(num, den)

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.h1, self.r_ref, self.r_new, self.h1c, self.R))


class FirstBlockCache:
    """State of one sampling run.  `threshold` (float >= 0, inf allowed) may be changed between steps.  `history` lists
    (indicator, skipped) for every forward since the last reset()."""

    def __init__(self, threshold):
        self.threshold = threshold
        self.reset()

    @property
    def threshold(self):
        return self._threshold

    @threshold.setter
    def threshold(self, value):
        self._threshold = check_threshold(value)

    def reset(self):
        """Drop all state and buffers: the next forward computes."""
        self.buffers = None
        self.has_state = False
        self.history = []

    def workspace(self, B, N, d, n_ref, n_seq, device):
        """The buffers of this geometry; a different key than the current one drops the state and the old buffers."""
        key = (int(B), int(N), int(d), int(n_ref), int(n_seq), torch.device(device))
        if self.buffers is None or self.buffers.key != key:
            self.buffers, self.has_state = None, False  # free the old set before allocating the new one
            self.buffers = Buffers(key)
        return self.buffers

    def decide(self, ind):
        """Skip iff there is state for the current buffers and ind < threshold.  Records (ind, skipped) in history."""
        skip = bool(self.has_state and ind < self._threshold)
        self.history.append((ind, skip))
        return skip

    def computed(self):
        """After a computed step: R holds its residual and r_new its r, which becomes r_ref (swap, no copy)."""
        b = self.buffers
        b.r_ref, b.r_new = b.r_new, b.r_ref
        self.has_state = True
