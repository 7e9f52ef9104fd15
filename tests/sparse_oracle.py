"""Test-side reference pieces for block-sparse self-attention: the dense key mask a tile map stands for, and fp32 softmax
attention under such a mask.  The model-level tests put masked_sdpa_fp32 in place of the oracle's self-attention sdpa
(oracle/dit_oracle.py itself has no mask)."""
import torch


def tile_mask(kv_tile_ptr, kv_tile_idx, q_len, kv_len, tile=128):
    """Expand a block-sparse map (query tile t attends to key tiles kv_tile_idx[kv_tile_ptr[t]:kv_tile_ptr[t+1]]) into a
    bool [q_len, kv_len] mask, True where a query may attend to a key."""
    ptr, idx = torch.as_tensor(kv_tile_ptr).long().cpu(), torch.as_tensor(kv_tile_idx).long().cpu()
    n_q, n_kv = ptr.numel() - 1, -(-kv_len // tile)
    rows = torch.repeat_interleave(torch.arange(n_q), ptr[1:] - ptr[:-1])
    tiles = torch.zeros(n_q, n_kv, dtype=torch.bool)
    tiles[rows, idx] = True
    return tiles.repeat_interleave(tile, 0).repeat_interleave(tile, 1)[:q_len, :kv_len]


def masked_sdpa_fp32(q, k, v, mask, chunk=512):
    """fp32 softmax(q k^T / sqrt(d)) v over the keys `mask` allows ([Lq, Lk] bool), queries chunked."""
    out = torch.empty_like(q)
    kt = k.transpose(-1, -2)
    for i in range(0, q.shape[-2], chunk):
        s = (q[..., i:i + chunk, :] @ kt) * q.shape[-1] ** -0.5
        out[..., i:i + chunk, :] = torch.softmax(s.masked_fill_(~mask[i:i + chunk], float("-inf")), -1) @ v
        del s
    return out
