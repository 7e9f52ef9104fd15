"""Content-adaptive block-sparse attention on the host: AdaptiveTiles validation, the model kwarg and its refusals, and the
selection rule (tests/adaptive_oracle.py, which the GPU tests hold the kernels to) on hand-made pooled tiles."""
import math

import numpy as np
import pytest
import torch

from adaptive_oracle import csr_to_dense, expand_rows, select_reference
from scail_b200 import ops, sparse

CFG = dict(hidden_size=128, num_attention_heads=1, inner_hidden_size=256, num_layers=2, text_dim=32, time_embed_dim=128)


# ---------------------------------------------------------------- AdaptiveTiles
@pytest.mark.parametrize("mass", [0, 0.0, 0.5, 0.9, 1, 1.0, np.float64(0.95)])
@pytest.mark.parametrize("cap", [None, 0, 3, np.int64(7)])
def test_adaptive_tiles_accepts_its_range(mass, cap):
    a = sparse.AdaptiveTiles(mass, cap)
    assert a.mass == float(mass) and type(a.mass) is float
    assert a.max_tiles == (None if cap is None else int(cap))
    assert a == sparse.AdaptiveTiles(float(mass), cap) and hash(a) == hash(sparse.AdaptiveTiles(float(mass), cap))


@pytest.mark.parametrize("mass", [-0.01, 1.01, math.nan, math.inf, True, False, "0.9", None, [0.9]])
def test_adaptive_tiles_refuses_bad_mass(mass):
    with pytest.raises(ValueError, match="mass"):
        sparse.AdaptiveTiles(mass)


@pytest.mark.parametrize("cap", [-1, 2.0, True, "3", 1.5])
def test_adaptive_tiles_refuses_bad_cap(cap):
    with pytest.raises(ValueError, match="max_tiles"):
        sparse.AdaptiveTiles(0.9, cap)


def test_scratch_length():
    assert ops.select_scratch_len(2, 40, 27904) == 2 * 40 * 218 * (1 + 7)
    assert ops.select_scratch_len(1, 1, 129) == 2 * (1 + 1)


# ---------------------------------------------------------------- the model kwarg
def test_model_kwarg_defaults_off_and_leaves_the_state_dict_alone():
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    a = DiffusionTransformer(attention_adaptive=sparse.AdaptiveTiles(0.9, 4), **CFG)
    torch.manual_seed(0)
    b = DiffusionTransformer(**CFG)
    assert a.mixins["adaln_layer"].attention_adaptive == sparse.AdaptiveTiles(0.9, 4)
    assert b.mixins["adaln_layer"].attention_adaptive is None
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)


@pytest.mark.parametrize("bad", [0.9, "0.9", 1, (0.9, 2)])
def test_model_kwarg_must_be_adaptive_tiles(bad):
    from scail_b200.dit import DiffusionTransformer
    with pytest.raises(ValueError, match="attention_adaptive"):
        DiffusionTransformer(attention_adaptive=bad, **CFG)


def test_window_and_adaptive_refused_together():
    from scail_b200.dit import DiffusionTransformer
    with pytest.raises(ValueError, match="attention_window and attention_adaptive"):
        DiffusionTransformer(attention_window=2, attention_adaptive=sparse.AdaptiveTiles(0.9), **CFG)
    m = DiffusionTransformer(attention_window=2, **CFG)
    ad = m.mixins["adaln_layer"]
    ad.attention_adaptive = sparse.AdaptiveTiles(0.9)  # toggled on as a plain attribute: refused at the next forward
    kw = dict(ref_length=16, seq_length=80, pose_length=20, rope_T=5, rope_H=4, rope_W=4)
    with pytest.raises(ValueError, match="attention_window and attention_adaptive"):
        ad._attention_tiles(torch.device("cpu"), 116, kw)


def test_context_parallel_refused():
    from scail_b200.dit import DiffusionTransformer

    class StubCP:
        size, rank = 2, 0

    m = DiffusionTransformer(attention_adaptive=sparse.AdaptiveTiles(0.5), **CFG)
    ad = m.mixins["adaln_layer"]
    ad.cp = StubCP()
    with pytest.raises(NotImplementedError, match="attention_adaptive"):
        ad._refuse_fp8_attention_cp()
    ad.attention_adaptive = None
    ad._refuse_fp8_attention_cp()  # off: nothing to refuse


# ---------------------------------------------------------------- the selection rule
def pooled(s_rows):
    """qbar, kbar [n, 128] whose scores s = qbar . kbar / sqrt(128) are the given [n, n] matrix (rank n <= 128)."""
    s = np.asarray(s_rows, np.float64)
    n = s.shape[0]
    q = np.zeros((n, 128))
    q[:, :n] = s * math.sqrt(128)
    k = np.zeros((n, 128))
    k[:, :n] = np.eye(n)
    return q, k


def test_rule_takes_the_largest_mass_first_and_stops_at_the_target():
    # query tile 0 of 5 full tiles, no ref: e = exp(s - max) over tiles [diag, 1, 2, 3, 4]
    s = np.zeros((5, 5))
    s[0] = [0.0, np.log(4), np.log(2), np.log(1), np.log(1)]  # e ~ [1, 4, 2, 1, 1] (times 128), total 9
    q, k = pooled(s)
    L = 5 * 128
    for mass, want in [(0.0, [0]), (0.1, [0]), (0.5, [0, 1]), (0.6, [0, 1, 2]), (0.75, [0, 1, 2]), (0.8, [0, 1, 2, 3]),
                       (0.95, [0, 1, 2, 3, 4]), (1.0, [0, 1, 2, 3, 4])]:
        listed, _ = select_reference(q, k, L, 0, mass)
        assert np.nonzero(listed[0])[0].tolist() == want, (mass, listed[0])


def test_rule_ties_go_to_the_lower_index_and_the_cap_counts_taken_tiles_only():
    s = np.zeros((6, 6))
    s[2] = [1.0, 3.0, 0.0, 3.0, 3.0, 1.0]  # tiles 1, 3, 4 tie
    q, k = pooled(s)
    L = 6 * 128
    listed, _ = select_reference(q, k, L, 0, 0.5)
    assert np.nonzero(listed[2])[0].tolist() == [1, 2, 3]  # diag 2, then 1 and 3 of the tie reach half the mass
    listed, _ = select_reference(q, k, L, 0, 0.99, max_tiles=2)
    assert np.nonzero(listed[2])[0].tolist() == [1, 2, 3]
    listed, _ = select_reference(q, k, L, 0, 1.0, max_tiles=0)
    assert np.nonzero(listed[2])[0].tolist() == [2]
    listed, _ = select_reference(q, k, L, 300, 1.0, max_tiles=1)  # ref tiles 0..2 forced; the cap adds one more
    assert np.nonzero(listed[2])[0].tolist() == [0, 1, 2, 3]


def test_rule_weights_the_ragged_last_tile_by_its_valid_keys():
    s = np.zeros((3, 3))
    s[0] = [0.0, 0.0, np.log(100.0)]  # the last tile scores 100x per key but holds 1 key: e = [128, 128, 100]
    q, k = pooled(s)
    listed, _ = select_reference(q, k, 2 * 128 + 1, 0, 0.5)
    assert np.nonzero(listed[0])[0].tolist() == [0, 1]  # 128 + 128 >= 0.5 * 356: the heavy ragged tile is not needed
    listed, _ = select_reference(q, k, 3 * 128, 0, 0.5)  # the same scores with a full last tile
    assert np.nonzero(listed[0])[0].tolist() == [0, 2]


def test_rule_forces_the_ref_and_diagonal_tiles_at_480x832():
    """480 x 832: 1560 ref tokens end inside tile 12 (not tile-aligned), so tiles 0..12 are forced for every query tile."""
    h, w, t = 60, 104, 21
    n_ref = (h // 2) * (w // 2)
    L = n_ref + t * n_ref + t * (h // 4) * (w // 4)
    n = -(-L // 128)
    assert n_ref % 128 != 0 and -(-n_ref // 128) == 13 and n == 333
    rng = np.random.default_rng(0)
    q, k = rng.standard_normal((2, n, 128)), rng.standard_normal((2, n, 128))
    listed, _ = select_reference(q, k, L, n_ref, 0.0)
    for hq in range(2):
        for r in range(n):
            want = sorted(set(range(13)) | {r})
            assert np.nonzero(listed[hq, r])[0].tolist() == want
    full, _ = select_reference(q, k, L, n_ref, 1.0)
    assert full.all()
    part, _ = select_reference(q, k, L, n_ref, 0.6)
    assert part[:, :, :13].all() and part[:, np.arange(n), np.arange(n)].all() and (part.sum(-1) >= 13).all()
    # monotone in the mass: a larger mass never drops a tile
    more, _ = select_reference(q, k, L, n_ref, 0.8)
    assert (more | ~part).all()


def test_near_flags_rows_at_the_cutoff():
    s = np.zeros((4, 4))
    s[0] = [0.0, 0.0, 0.0, 0.0]  # e = 128 each, total 512: mass 0.5 is met exactly after one taken tile
    q, k = pooled(s)
    _, near = select_reference(q, k, 512, 0, 0.5, band=1e-5)
    assert near[0]
    _, near = select_reference(q, k, 512, 0, 0.4, band=1e-5)
    assert near[0]  # ties between the last taken and the first dropped tile


def test_expand_rows_matches_the_tile_mask():
    from sparse_oracle import tile_mask
    ptr = np.array([0, 2, 3, 6])
    idx = np.array([0, 2, 1, 0, 1, 2])
    L = 300
    tm = torch.from_numpy(csr_to_dense(ptr, idx, 3))[None, None]
    want = tile_mask(ptr, idx, L, L)
    for i0, i1 in [(0, 300), (0, 128), (128, 300), (256, 300)]:
        assert torch.equal(expand_rows(tm, i0, i1, L)[0, 0], want[i0:i1])
