"""Test-side restatement of the first-block residual cache (scail_b200.step_cache): the model's own hooks (patch embedding,
layer_forward, final_forward) for the network, and torch fp32 / fp64 arithmetic for everything the cache's kernels do."""
import math

import torch


def indicator_sums(h0, h1, r_ref, chunk=1 << 24):
    """(r = bf16(f32(h1) - f32(h0)), sum|r - r_ref|, sum|r_ref|) with the sums in fp64 (chunked, for 14B-width tensors)."""
    r = torch.empty_like(h1)
    num = den = 0.0
    a, b, c, o = h0.reshape(-1), h1.reshape(-1), r_ref.reshape(-1), r.view(-1)
    for i in range(0, a.numel(), chunk):
        s = slice(i, i + chunk)
        o[s] = (b[s].float() - a[s].float()).to(torch.bfloat16)
        num += float((o[s].double() - c[s].double()).abs().sum())
        den += float(c[s].double().abs().sum())
    return r, num, den


def update_ref(h, h1c, n_ref):
    n_seq = h1c.shape[1]
    return h[:, n_ref:n_ref + n_seq].float() - h1c.float()


def apply_ref(h, R, n_ref):
    out = h.clone()
    rows = out[:, n_ref:n_ref + R.shape[1]]
    rows.copy_((rows.float() + R).to(torch.bfloat16))
    return out


class RestatedCache:
    """The cache's semantics over whole forwards: forward(threshold, x, **model kwargs) -> the velocity, with
    history = [(indicator, skipped)] as FirstBlockCache keeps it."""

    def __init__(self, model):
        self.m = model
        self.r_ref = self.R = None
        self.history = []

    def forward(self, threshold, x, timesteps=None, context=None, **kwargs):
        m = self.m
        ad, fl = m.mixins["adaln_layer"], m.mixins["final_layer"]
        h0, kw, _ = m._tokens(x, timesteps, context, None, dict(kwargs))
        h0 = h0.clone()
        h1 = ad.layer_forward(h0.clone(), None, layer_id=0, **kw).clone()
        n_ref, n_seq = kw["ref_length"], kw["seq_length"]
        r, num, den = indicator_sums(h0, h1, self.r_ref if self.r_ref is not None else torch.zeros_like(h1))
        ind = math.inf if den == 0 else num / den
        skip = self.r_ref is not None and ind < threshold
        self.history.append((ind, skip))
        if skip:
            h = apply_ref(h1, self.R, n_ref)
        else:
            h = h1.clone()
            for l in range(1, m.num_layers):
                h = ad.layer_forward(h, None, layer_id=l, **kw)
            self.R = update_ref(h, h1[:, n_ref:n_ref + n_seq], n_ref)
            self.r_ref = r
        return fl.final_forward(h, **kw)
