"""Test-side restatement of content-adaptive tile selection (scail_b200.sparse.AdaptiveTiles, select_tiles_kernel) in
float64 numpy, and fp32 softmax attention under per-(batch, head) tile masks."""
import numpy as np

TILE = 128


def select_reference(qbar, kbar, L, n_ref, mass, max_tiles=None, band=0.0, tie_band=1e-9):
    """The selection rule on pooled tiles qbar, kbar [..., n, 128] (float64 arithmetic):
    s = qbar_q . kbar_k / sqrt(128), e_k = n_k exp(s_k - max_k s), n_k the valid keys of tile k.  Forced: k == q and every
    k < ceil(n_ref / 128).  The others by e descending (ties: lower k) until the forced plus taken sum reaches mass * sum(e),
    or max_tiles were taken; mass >= 1 takes every tile up to the cap.  Sums run in ascending order (as the kernel's).
    -> (listed bool [..., n, n], near bool [..., n]): near marks rows whose decision may flip under rounding: a partial sum
    next to the cutoff within band * sum(e) of the target, or the last taken and the first dropped e within a relative
    tie_band of each other (the kernel's fp64 sums run in another order than numpy's)."""
    qb, kb = np.asarray(qbar, np.float64), np.asarray(kbar, np.float64)
    n = qb.shape[-2]
    s = (qb @ np.swapaxes(kb, -1, -2)) * 128 ** -0.5
    nk = np.minimum(TILE, L - TILE * np.arange(n)).astype(np.float64)
    e = nk * np.exp(s - s.max(-1, keepdims=True))
    n_ref_t = -(-int(n_ref) // TILE)
    listed = np.zeros(e.shape, dtype=bool)
    near = np.zeros(e.shape[:-1], dtype=bool)
    for ix in np.ndindex(*e.shape[:-1]):
        q, ei = ix[-1], e[ix]
        forced = np.zeros(n, dtype=bool)
        forced[:n_ref_t] = True
        forced[q] = True
        total = np.cumsum(ei)[-1]
        cum = np.cumsum(ei[forced])[-1]
        free = np.nonzero(~forced)[0]
        order = free[np.lexsort((free, -ei[free]))]
        cap = free.size if max_tiles is None else min(int(max_tiles), free.size)
        if mass >= 1.0:
            m = cap
        else:
            target = mass * total
            sums = [cum]
            m = 0
            while m < cap and cum < target:
                cum += ei[order[m]]
                m += 1
                sums.append(cum)
            # mass 0: the forced sum is >= 0 = target exactly, so nothing can flip
            near[ix] = mass > 0 and any(abs(x - target) <= band * total for x in sums[-2:])
            if 0 < m < free.size and abs(ei[order[m - 1]] - ei[order[m]]) <= tie_band * ei[order[m - 1]]:
                near[ix] = True
        row = listed[ix]
        row[forced] = True
        row[order[:m]] = True
    return listed, near


def csr_to_dense(ptr, idx, n):
    """One CSR map -> bool [n, n]."""
    m = np.zeros((n, n), dtype=bool)
    m[np.repeat(np.arange(n), np.diff(ptr)), idx] = True
    return m


def expand_rows(tmask, i0, i1, L):
    """Token mask rows [i0, i1) of per-(batch, head) tile masks tmask bool [B, H, n, n] (torch) -> bool [B, H, i1 - i0, L]."""
    t = tmask[:, :, i0 // TILE:-(-i1 // TILE)].repeat_interleave(TILE, 2)
    t = t[:, :, i0 - (i0 // TILE) * TILE:][:, :, :i1 - i0]
    return t.repeat_interleave(TILE, 3)[..., :L]


def masked_sdpa_bh(q, k, v, tmask, chunk=512):
    """fp32 softmax(q k^T / sqrt(d)) v, q, k, v [B, H, L, D], each (b, h) over the key tiles tmask[b, h] lists for the
    query's tile.  chunk must be a multiple of 128."""
    import torch
    out = torch.empty_like(q)
    L = q.shape[-2]
    kt = k.transpose(-1, -2)
    for i in range(0, L, chunk):
        j = min(L, i + chunk)
        s = (q[..., i:j, :] @ kt) * q.shape[-1] ** -0.5
        out[..., i:j, :] = torch.softmax(s.masked_fill_(~expand_rows(tmask, i, j, L), float("-inf")), -1) @ v
        del s
    return out
