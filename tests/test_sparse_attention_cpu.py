"""Frame-window block-sparse attention on the host: the tile map's format and policy (scail_b200.sparse), its densities at
the three standard resolutions, the ops wrapper's validation of malformed maps, the model kwarg and the test-side reference mask."""
import numpy as np
import pytest
import torch

from scail_b200 import ops, sparse

T = 21
# (latent h, w) -> density at windows 1, 2, 3, 5 (tile pairs listed / all tile pairs)
DENSITY = {(64, 64): (218, [0.2004, 0.2804, 0.3561, 0.4950]),    # 512 x 512
           (64, 112): (382, [0.2025, 0.2822, 0.3578, 0.4963]),   # 512 x 896
           (60, 104): (333, [0.2195, 0.2983, 0.3727, 0.5090])}   # 480 x 832: segments not tile-aligned


def geometry(h, w, t=T):
    H, W = h // 2, w // 2
    return sparse.geometry(ref_length=H * W, seq_length=t * H * W, pose_length=t * (h // 2) * (w // 2) // 4, rope_T=t,
                           rope_H=H, rope_W=W)


def dense(ptr, idx):
    n = ptr.size - 1
    m = np.zeros((n, n), dtype=bool)
    m[np.repeat(np.arange(n), np.diff(ptr)), idx] = True
    return m


@pytest.mark.parametrize("hw", list(DENSITY))
@pytest.mark.parametrize("window", [0, 1, 2, 3, 5])
def test_map_format_and_policy(hw, window):
    g = geometry(*hw)
    ptr, idx, density = sparse.frame_window_tiles(g, window)
    n = DENSITY[hw][0]
    assert ptr.dtype == np.int32 and idx.dtype == np.int32 and ptr.shape == (n + 1,) and ptr[0] == 0 and ptr[-1] == idx.size
    for q in range(n):
        row = idx[ptr[q]:ptr[q + 1]]
        assert row.size > 0 and (np.diff(row) > 0).all() and row.min() >= 0 and row.max() < n
    m = dense(ptr, idx)
    assert (m == m.T).all()  # symmetric
    n_ref_tiles = -(-g.ref_length // 128)
    assert m[:n_ref_tiles].all()        # (a) the ref query rows are dense
    assert m[:, :n_ref_tiles].all()     # (b) every row lists every ref key tile
    assert density == idx.size / n ** 2
    # (c) at token level: a query and a key of two frames within the window always meet
    lab = np.full(n * 128, -1)
    tok = np.arange(g.ref_length + g.seq_length + g.pose_length)
    noise = (tok >= g.ref_length) & (tok < g.ref_length + g.seq_length)
    lab[tok[noise]] = (tok[noise] - g.ref_length) // (g.H * g.W)
    pose = tok >= g.ref_length + g.seq_length
    lab[tok[pose]] = (tok[pose] - g.ref_length - g.seq_length) // ((g.H // 2) * (g.W // 2))
    for f in range(T):
        for f2 in range(max(0, f - window), min(T, f + window + 1)):
            qt = np.unique(np.nonzero(lab == f)[0] // 128)
            kt = np.unique(np.nonzero(lab == f2)[0] // 128)
            assert m[np.ix_(qt, kt)].all()


@pytest.mark.parametrize("hw", list(DENSITY))
def test_densities_match_the_table(hw):
    g = geometry(*hw)
    n, want = DENSITY[hw]
    got = [round(sparse.frame_window_tiles(g, w)[2], 4) for w in (1, 2, 3, 5)]
    assert got == want
    assert sparse.frame_window_tiles(g, 0)[2] < want[0]


@pytest.mark.parametrize("hw", list(DENSITY))
def test_window_of_t_minus_1_is_the_full_map(hw):
    g = geometry(*hw)
    n = DENSITY[hw][0]
    for w in (T - 1, T, 100):
        ptr, idx, density = sparse.frame_window_tiles(g, w)
        assert density == 1.0 and np.array_equal(idx, np.tile(np.arange(n), n))
    assert sparse.frame_window_tiles(g, T - 2)[2] < 1.0


def test_geometry_and_window_are_checked():
    with pytest.raises(ValueError, match="layout"):
        sparse.geometry(ref_length=64, seq_length=3 * 64, pose_length=40, rope_T=3, rope_H=8, rope_W=8)
    g = geometry(16, 16, 3)
    for bad in (-1, 1.5, "2", True):
        with pytest.raises(ValueError, match="attention_window"):
            sparse.frame_window_tiles(g, bad)


def _ok_map():
    # L = 600: 5 tiles, the last ragged
    return np.array([0, 1, 3, 6, 8, 13]), np.array([4, 0, 2, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])


MALFORMED = {
    "empty row": (np.array([0, 1, 1, 4, 6, 11]), np.array([4, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "descending row": (np.array([0, 1, 3, 6, 8, 13]), np.array([4, 2, 0, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "repeated tile": (np.array([0, 1, 3, 6, 8, 13]), np.array([4, 0, 0, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "index past the last key tile": (np.array([0, 1, 3, 6, 8, 13]), np.array([5, 0, 2, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "negative index": (np.array([0, 1, 3, 6, 8, 13]), np.array([-1, 0, 2, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "too few rows": (np.array([0, 1, 3, 6, 8]), np.array([4, 0, 2, 0, 1, 4, 3, 4])),
    "ptr does not end at nnz": (np.array([0, 1, 3, 6, 8, 12]), np.array([4, 0, 2, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "ptr does not start at 0": (np.array([1, 1, 3, 6, 8, 13]), np.array([4, 0, 2, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4])),
    "float indices": (np.array([0, 1, 3, 6, 8, 13]), np.array([4, 0, 2, 0, 1, 4, 3, 4, 0, 1, 2, 3, 4], dtype=np.float32)),
}


@pytest.mark.parametrize("what", list(MALFORMED))
def test_ops_wrapper_rejects_malformed_maps(what):
    ptr, idx = MALFORMED[what]
    L = 600
    t = torch.zeros(L, 128, dtype=torch.bfloat16)  # CPU tensors: the map is checked before anything needs a GPU
    with pytest.raises(ValueError, match="tile map"):
        ops.attention_sparse(t, t, t, t, 1, 1, L, (torch.from_numpy(ptr), torch.from_numpy(idx)))
    with pytest.raises(ValueError, match="tile map"):
        ops.attention_fp8_sparse(t, t, t, t, t, t, t, 1, 1, L, (ptr, idx))
    with pytest.raises(ValueError, match="tile map"):
        ops.TileMap(ptr, idx, L, L)


def test_a_valid_map_passes_validation_and_then_needs_cuda():
    ptr, idx = _ok_map()
    m = ops.TileMap(ptr, idx, 600, 600)
    assert (m.n_q_tiles, m.n_kv_tiles, m.nnz) == (5, 5, 13) and m.density == 13 / 25
    with pytest.raises(ValueError, match="tile map"):  # a valid map for another length
        ops.TileMap(ptr, idx, 700, 700)
    t = torch.zeros(600, 128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.attention_sparse(t, t, t, t, 1, 1, 600, m)


def test_model_kwarg_defaults_off_and_leaves_the_state_dict_alone():
    from scail_b200.dit import DiffusionTransformer
    cfg = dict(hidden_size=128, num_attention_heads=1, inner_hidden_size=256, num_layers=2, text_dim=32, time_embed_dim=128)
    torch.manual_seed(0)
    a = DiffusionTransformer(attention_window=2, **cfg)
    torch.manual_seed(0)
    b = DiffusionTransformer(**cfg)
    assert a.mixins["adaln_layer"].attention_window == 2 and b.mixins["adaln_layer"].attention_window is None
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    with pytest.raises(ValueError, match="attention_window"):
        DiffusionTransformer(attention_window=-1, **cfg)


def test_reference_mask_expands_the_map_and_masks_the_softmax():
    from oracle import dit_oracle as O
    from sparse_oracle import masked_sdpa_fp32, tile_mask
    ptr, idx = _ok_map()
    mask = tile_mask(ptr, idx, 600, 600)
    assert mask.shape == (600, 600)
    assert mask[:128, 512:].all() and not mask[:128, :512].any()  # query tile 0: only the ragged last key tile
    assert mask[512:].all()  # query tile 4 lists every key tile
    g = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(1, 1, 600, 16, generator=g) for _ in range(3))
    got = masked_sdpa_fp32(q, k, v, mask, chunk=256)
    want = O.sdpa(q[:, :, :128], k[:, :, 512:], v[:, :, 512:])
    assert torch.allclose(got[:, :, :128], want, atol=1e-6)
    full = masked_sdpa_fp32(q, k, v, torch.ones(600, 600, dtype=torch.bool))
    assert torch.allclose(full, O.sdpa(q, k, v), atol=1e-6)
