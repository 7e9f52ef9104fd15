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
tile (the dense map).

The module also holds the content-adaptive policy (AdaptiveTiles): per forward, per layer and per (batch, head), each query
tile keeps the key tiles that carry a chosen share of the softmax mass estimated from tile-pooled Q and K, always with its
diagonal tile and the tiles holding reference tokens.  Those maps are chosen on the device (ops.tile_pool,
ops.select_tiles) and run through the per-(batch, head) sparse kernels."""
import math
import numbers
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


# ---------------------------------------------------------------- content-adaptive tiles
RECORD = None  # a list to collect (kv_tile_ptr, kv_tile_idx) copies of every map AdaptiveTiles.select builds (tests)


class AdaptiveTiles:
    """Content-adaptive block-sparse self-attention.  mass in [0, 1]: per query tile, the key tiles are listed by estimated
    softmax mass e_k = n_k exp(s_k - max s), s_k = mean(Q over the query tile) . mean(K over key tile k) / sqrt(128), n_k the
    valid keys of tile k, until the listed share of sum_k e_k reaches `mass` (1: every tile; 0: only the forced tiles, the
    diagonal tile and those holding reference tokens).  max_tiles: None, or an int >= 0 capping the tiles taken by mass
    (forced tiles do not count).  1 - mass estimates the attention mass dropped; it says nothing about visual quality."""

    def __init__(self, mass, max_tiles=None):
        if isinstance(mass, bool) or not isinstance(mass, numbers.Real) or math.isnan(float(mass)) or not 0.0 <= float(mass) <= 1.0:
            raise ValueError(f"AdaptiveTiles: mass must be a float in [0, 1], got {mass!r}")
        if max_tiles is not None and (isinstance(max_tiles, bool) or not isinstance(max_tiles, (int, np.integer)) or
                                      max_tiles < 0):
            raise ValueError(f"AdaptiveTiles: max_tiles must be None or an int >= 0, got {max_tiles!r}")
        self.mass = float(mass)
        self.max_tiles = None if max_tiles is None else int(max_tiles)

    def __repr__(self):
        return f"AdaptiveTiles(mass={self.mass!r}, max_tiles={self.max_tiles!r})"

    def __eq__(self, other):
        return isinstance(other, AdaptiveTiles) and (self.mass, self.max_tiles) == (other.mass, other.max_tiles)

    def __hash__(self):
        return hash((self.mass, self.max_tiles))

    def select(self, q, k, B, H, L, n_ref, buf, q_scale=None, k_scale=None):
        """Pool the self-attention operands q, k ([B*L, H*128] slabs: bf16, or e4m3 with their [B, H, L_pad] scales) and
        choose this forward's maps on the device.  buf(name, shape, dtype) supplies the buffers (the model's per-stream
        workspace, so a captured graph reads fixed addresses).  -> (kv_tile_ptr int32 [B, H, n + 1], kv_tile_idx int32
        [B, H, n * n]) for ops.attention_sparse_bh / attention_fp8_sparse_bh."""
        import torch
        n = -(-int(L) // TILE)
        f32, i32 = torch.float32, torch.int32
        qbar = ops.tile_pool(q, B, H, L, buf("ada_qbar", (B, H, n, 128), f32), x_scale=q_scale)
        kbar = ops.tile_pool(k, B, H, L, buf("ada_kbar", (B, H, n, 128), f32), x_scale=k_scale)
        ptr, idx = buf("ada_ptr", (B, H, n + 1), i32), buf("ada_idx", (B, H, n * n), i32)
        ops.select_tiles(qbar, kbar, B, H, L, n_ref, self.mass, self.max_tiles, ptr, idx,
                         buf("ada_scratch", (ops.select_scratch_len(B, H, L),), i32))
        if RECORD is not None:
            RECORD.append((ptr.clone(), idx.clone()))
        return ptr, idx


def check_adaptive(adaptive):
    """The attention_adaptive setting: None or an AdaptiveTiles."""
    if adaptive is not None and not isinstance(adaptive, AdaptiveTiles):
        raise ValueError(f"attention_adaptive must be None or a scail_b200.sparse.AdaptiveTiles, got {adaptive!r}")
    return adaptive


def bh_maps_host(ptr, idx):
    """Per-(batch, head) device maps -> {(b, h): (kv_tile_ptr, kv_tile_idx)} numpy int32, each trimmed to its own nnz."""
    p, i = ptr.cpu().numpy(), idx.cpu().numpy()
    return {(b, h): (p[b, h].copy(), i[b, h, :p[b, h, -1]].copy()) for b in range(p.shape[0]) for h in range(p.shape[1])}
