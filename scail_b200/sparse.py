"""Opt-in block-sparse self-attention: the frame-window mask over SCAIL's ref || noise || pose token layout.

This module is the only place that knows the mask policy.  The kernels (scail_attention_sparse, scail_attention_fp8_sparse)
take a generic tile map: for each 128-row query tile a CSR row of 128-key tiles (ops.TileMap), and compute exact softmax
attention over every key of the listed tiles.

Labels.  Ref tokens [0, n_ref) carry the label R.  Noise token i is in frame (i - n_ref) // (H' W') and pose token i in
frame (i - n_ref - n_noise) // (H'/2 W'/2), with H' x W' the token grid (rope_H x rope_W).  A tile carries the labels of its
tokens.  Key tile k is listed for query tile q when
  (a) q holds a ref token (the ref rows stay dense), or
  (b) k holds a ref token (every query sees the whole reference image), or
  (c) some frame of q and some frame of k differ by at most `window`, a tile's frames being the span from its lowest to
      its highest frame (see frame_window_tiles).
A tile that straddles a segment or frame boundary therefore takes part with all its tokens.  window >= T - 1 lists every
tile (the dense map)."""
import threading
from collections import namedtuple

import numpy as np

from . import ops

TILE = 128

Geometry = namedtuple("Geometry", "ref_length seq_length pose_length T H W")
Geometry.__doc__ = "Token layout of one SCAIL sequence: segment lengths and the T x H' x W' token grid of the noise segment."


def geometry(ref_length, seq_length, pose_length, rope_T, rope_H, rope_W, **_):
    """The Geometry of the forward kwargs DiffusionTransformer.forward builds (extra keys are ignored)."""
    g = Geometry(int(ref_length), int(seq_length), int(pose_length), int(rope_T), int(rope_H), int(rope_W))
    if g.T < 1 or g.ref_length != g.H * g.W or g.seq_length != g.T * g.H * g.W or \
            g.pose_length != g.T * (g.H // 2) * (g.W // 2):
        raise ValueError(f"frame-window attention: inconsistent token layout {g}")
    return g


def check_window(window):
    if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or window < 0:
        raise ValueError(f"attention_window must be None or an int >= 0, got {window!r}")
    return int(window)


def tile_frames(g):
    """(has_ref, lo, hi), each [n_tiles]: whether a 128-token tile holds a ref token, and the lowest and highest frame of its
    noise and pose tokens (lo > hi for a tile without any)."""
    n = g.ref_length + g.seq_length + g.pose_length
    n_tiles = (n + TILE - 1) // TILE
    tok = np.arange(n_tiles * TILE)
    frame = np.full(tok.shape, -1)
    noise = (tok >= g.ref_length) & (tok < g.ref_length + g.seq_length)
    frame[noise] = (tok[noise] - g.ref_length) // (g.H * g.W)
    pose = (tok >= g.ref_length + g.seq_length) & (tok < n)
    frame[pose] = (tok[pose] - g.ref_length - g.seq_length) // ((g.H // 2) * (g.W // 2))
    frame = frame.reshape(n_tiles, TILE)
    has_ref = (tok.reshape(n_tiles, TILE) < g.ref_length).any(1)
    lo = np.where(frame >= 0, frame, g.T).min(1)
    hi = frame.max(1)
    return has_ref, lo, hi


def frame_window_tiles(g, window):
    """The frame-window map of geometry g on the host: (kv_tile_ptr int32 [n_tiles + 1], kv_tile_idx int32 [nnz], density),
    density = listed tile pairs / all tile pairs, exactly.  The map is validated (ops.check_tile_map) before it is returned.

    A tile's frames are taken as the whole span [lo, hi] of its noise and pose frames.  Where segments are tile-aligned
    (512 x 512, 512 x 896) that is exactly the set of its frames.  The one tile that straddles the noise -> pose boundary
    otherwise (e.g. 480 x 832) holds noise frame T - 1 and pose frame 0; its span covers every frame, so its row and column
    are dense.  The map is then a superset of the per-frame rule: it never drops a key a frame within `window` would keep."""
    window = check_window(window)
    has_ref, lo, hi = tile_frames(g)
    n_tiles = has_ref.size
    near = (lo[:, None] - window <= hi[None, :]) & (lo[None, :] - window <= hi[:, None])
    listed = near | has_ref[:, None] | has_ref[None, :]
    ptr = np.zeros(n_tiles + 1, dtype=np.int32)
    ptr[1:] = np.cumsum(listed.sum(1))
    idx = np.nonzero(listed)[1].astype(np.int32)  # row-major: each row's columns ascending
    n = g.ref_length + g.seq_length + g.pose_length
    ops.check_tile_map(ptr, idx, n, n)
    return ptr, idx, idx.size / float(n_tiles * n_tiles)


_CACHE = {}
_LOCK = threading.Lock()


def tile_map(g, window, device):
    """The uploaded ops.TileMap of frame_window_tiles(g, window) on `device`, built once per (geometry, window, device) and
    kept for the life of the process, so its tensors stay at fixed addresses (a captured CUDA graph reads them)."""
    import torch
    window = check_window(window)
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    key = (g, window, str(device))
    with _LOCK:
        m = _CACHE.get(key)
        if m is None:
            ptr, idx, density = frame_window_tiles(g, window)
            n = g.ref_length + g.seq_length + g.pose_length
            m = ops.TileMap(ptr, idx, n, n, device=device, checked=True)
            m.density = density
            _CACHE[key] = m
    return m
