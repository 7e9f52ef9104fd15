"""CPU tests of the chunked VAE decode / encode: argument checks, no CPU path, and the chunk / frame planning."""
import pytest
import torch


def test_chunk_frames_must_be_positive():
    from scail_b200.wan_vae import WanVAE, chunk_ranges
    v = WanVAE(dim=16, device="cpu")
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            v.decode([torch.zeros(16, 2, 4, 4)], chunk_frames=bad)
        with pytest.raises(ValueError):
            v.encode([torch.zeros(3, 5, 32, 32)], chunk_frames=bad)
        with pytest.raises(ValueError):
            chunk_ranges(5, bad)
    with pytest.raises(ValueError):
        WanVAE(dim=16, device="cpu", chunk_frames=0)


def test_chunked_paths_have_no_cpu_fallback():
    from scail_b200.wan_vae import WanVAE
    v = WanVAE(dim=16, device="cpu", chunk_frames=2)
    with pytest.raises(RuntimeError, match="no CPU path"):
        v.decode([torch.zeros(16, 3, 4, 4)])
    with pytest.raises(RuntimeError, match="no CPU path"):
        v.encode([torch.zeros(3, 9, 32, 32)])
    with pytest.raises(RuntimeError, match="no CPU path"):
        v.decode([torch.zeros(16, 3, 4, 4)], chunk_frames=1)


def test_chunk_ranges_cover_the_latent_frames():
    from scail_b200.wan_vae import chunk_ranges
    assert chunk_ranges(5, 1) == [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5)]
    assert chunk_ranges(5, 2) == [(0, 2), (2, 4), (4, 5)]
    assert chunk_ranges(5, 3) == [(0, 3), (3, 5)]
    assert chunk_ranges(5, 8) == [(0, 5)]
    assert chunk_ranges(21, 4)[-1] == (20, 21)


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_frame_ranges_per_stage(k):
    """Decode stages are 1+2(k-1) / 2k frames (x2) and 1+4(k-1) / 4k (x4, pixels); encode chunks are the same pixel ranges,
    k = 1 being the reference's 1, 4, 4, ... split.  The ranges of consecutive chunks tile the whole sequence."""
    from scail_b200.wan_vae import chunk_ranges, frame_range
    n = 7
    for up in (1, 2, 4):
        ranges = [frame_range(a, b, up) for a, b in chunk_ranges(n, k)]
        assert ranges[0][0] == 0 and ranges[-1][1] == 1 + up * (n - 1)
        assert all(r0[1] == r1[0] for r0, r1 in zip(ranges, ranges[1:]))
        assert ranges[0][1] - ranges[0][0] == 1 + up * (k - 1)
        for (a, b), (p0, p1) in zip(chunk_ranges(n, k)[1:], ranges[1:]):
            assert p1 - p0 == up * (b - a)
    assert [frame_range(a, b, 4) for a, b in chunk_ranges(3, 1)] == [(0, 1), (1, 5), (5, 9)]


def test_history_keeps_last_frames():
    from scail_b200.wan_vae import _History
    h = _History(2)
    assert h.frames() is None
    h.keep(torch.tensor([[1.0]]))
    assert h.frames().tolist() == [[1.0]]
    ptr = h.buf.data_ptr()
    h.keep(torch.tensor([[2.0]]))
    assert h.frames().tolist() == [[1.0], [2.0]]
    h.keep(torch.tensor([[3.0]]))
    assert h.frames().tolist() == [[2.0], [3.0]]
    h.keep(torch.tensor([[4.0], [5.0], [6.0]]))
    assert h.frames().tolist() == [[5.0], [6.0]] and h.buf.data_ptr() == ptr
    h1 = _History(1)
    h1.keep(torch.tensor([[1.0], [2.0]]))
    h1.keep(torch.tensor([[3.0]]))
    assert h1.frames().tolist() == [[3.0]]
