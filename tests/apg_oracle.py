"""APG (Sadat, Hilliges, Weber, ICLR 2025) restated in plain torch fp64, independent of scail_b200: one guided step of the
rule scail_b200.guidance states, per latent frame x[0, t]."""
import torch


def apg_parts(x, u, c, sigma, scale, eta, norm_threshold=0.0, momentum=0.0, avg=None):
    """Every piece of one step in fp64, from the latent x [1, T, ...] and the CFG pair (u, c) of its shape.  avg is the
    momentum average before the step (None: zero).  -> dict of D_c, diff (after momentum and threshold), par, orth, D_g,
    avg (after the step; None without momentum), f [T] (threshold factor) and p [T] (projection coefficient of diff)."""
    x, u, c = (t.double() for t in (x, u, c))
    dc = x - sigma * c
    diff = dc - (x - sigma * u)
    new_avg = None
    if momentum != 0.0:
        new_avg = diff + momentum * (torch.zeros_like(diff) if avg is None else avg.double())
        diff = new_avg
    T = x.shape[1]
    d, pc = diff.reshape(T, -1), dc.reshape(T, -1)
    norm = d.norm(dim=1)
    f = torch.ones_like(norm)
    if norm_threshold > 0.0:
        f = torch.where(norm > norm_threshold, norm_threshold / norm, f)
    d = d * f[:, None]
    nc = (pc * pc).sum(1)
    p = torch.where(nc == 0, torch.zeros_like(nc), (d * pc).sum(1) / nc)
    par = p[:, None] * pc
    orth = d - par
    dg = pc + (scale - 1.0) * (orth + eta * par)
    shape = x.shape
    return dict(D_c=dc, diff=d.view(shape), par=par.view(shape), orth=orth.view(shape), D_g=dg.view(shape), avg=new_avg,
                f=f, p=p)


def euler(x, d_g, sigma, next_sigma):
    """x' = x + (sigma' - sigma) (x - D_g) / sigma, in fp64."""
    x = x.double()
    return x + (next_sigma - sigma) * (x - d_g.double()) / sigma


def vanilla_cfg_euler(x, u, c, scale, sigma, next_sigma):
    """The sampler's vanilla step x + (sigma' - sigma) (u + s (c - u)), in fp64."""
    x, u, c = (t.double() for t in (x, u, c))
    return x + (next_sigma - sigma) * (u + scale * (c - u))
