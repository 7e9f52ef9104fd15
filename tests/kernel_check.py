"""Strict comparison of a kernel result with a high-precision reference of the same operation.

rel-L2 alone cannot see a localized error in a large tensor: one 2x512x896x96 output has 88 M elements, and one pixel
whose 96 channels are all wrong moves rel-L2 by about sqrt(96 / 88M) ~ 1e-3.  A halo or tap bug confined to an edge
column or a corner tile is exactly that kind of error.  So `assert_close_bf16` also bounds every element:

    |got - want| <= 2^-8 * |want| + 2^-12 * max|want|

bf16 carries 8 significant bits, so rounding an fp32 value once to nearest moves it by at most half an ulp, 2^-8 of its
magnitude (8.031 -> 8.0 is that worst case).  The relative term is therefore exactly one rounding, and a second rounding
anywhere in the chain can exceed it.  The absolute term is the slack for the kernel's fp32 accumulator differing from the
reference's (summation order, approximate exp / rsqrt): those differences are ~1e-6 of the terms, far below 2^-12 of the
largest output.  Composite results (several bf16 roundings in a chain) pass looser `elem_rel` / `elem_abs` and say why at
the call.

Everything is computed on the tensors' own device (no copy to the host), in fp32."""
from collections import namedtuple

import torch

ELEM_REL = 2.0 ** -8
ELEM_ABS = 2.0 ** -12

Check = namedtuple("Check", "rel_l2 worst_ratio n_bad worst_index got_at_worst want_at_worst bound_at_worst")


def measure(got, want, elem_rel=ELEM_REL, elem_abs=ELEM_ABS):
    """Compare got with want (same shape).  worst_ratio = max |got - want| / bound over all elements (> 1 fails the
    elementwise bound); worst_index is that element's index in the tensor's own shape.  NaN / inf count as violations.
    Neither got nor want is modified."""
    assert got.shape == want.shape, (tuple(got.shape), tuple(want.shape))
    want = want.float()
    d = got.to(torch.float32, copy=True).sub_(want)  # a copy even when got is fp32: the in-place ops below
    rel = float(d.norm().double() / want.norm().double())
    d.abs_()
    bound = want.abs()
    floor = elem_abs * float(bound.max())
    bound.mul_(elem_rel).add_(floor)
    ok = d <= bound  # False for NaN
    n_bad = int(ok.numel() - ok.sum())
    ratio = d.div_(bound.clamp_min_(torch.finfo(torch.float32).tiny)).nan_to_num_(nan=float("inf"))
    flat = int(ratio.argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), tuple(got.shape)))
    g, w = float(got.reshape(-1)[flat]), float(want.reshape(-1)[flat])
    return Check(rel, float(ratio.reshape(-1)[flat]), n_bad, idx, g, w, elem_rel * abs(w) + floor)


def assert_close_bf16(got, want, what, rel_l2=4e-3, elem_rel=ELEM_REL, elem_abs=ELEM_ABS):
    """Assert rel-L2(got, want) <= rel_l2 and the elementwise bound above.  Returns the Check for printing."""
    c = measure(got, want, elem_rel, elem_abs)
    where = (f"worst element at {c.worst_index} of shape {tuple(got.shape)}: got {c.got_at_worst:.6g}, want "
             f"{c.want_at_worst:.6g}, bound {c.bound_at_worst:.3g} (|diff| / bound = {c.worst_ratio:.3g})")
    assert c.n_bad == 0, (f"{what}: {c.n_bad} of {got.numel()} elements exceed |d| <= {elem_rel:.3g}|want| + "
                          f"{elem_abs:.3g} max|want| (rel-L2 {c.rel_l2:.3e}); {where}")
    assert c.rel_l2 <= rel_l2, f"{what}: rel-L2 {c.rel_l2:.3e} > {rel_l2:.1e}; {where}"
    return c
