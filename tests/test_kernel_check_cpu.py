"""kernel_check.assert_close_bf16 on the CPU: a once-rounded bf16 result passes, and one wrong pixel in a large
channels-last tensor fails it although rel-L2 alone would let it through (the reason the elementwise bound exists)."""
import pytest
import torch

from kernel_check import assert_close_bf16, measure


def test_once_rounded_bf16_passes():
    g = torch.Generator().manual_seed(0)
    want = torch.randn(3, 17, 40, 96, generator=g) * 3
    want[0, 0, 0] = 0  # exact zeros and values far below max|want| are covered by the absolute term
    want[1, 2, 3] *= 1e-6
    c = assert_close_bf16(want.to(torch.bfloat16), want, "once-rounded")
    # half a bf16 ulp reaches 2^-8 |want| just above a power of two: the relative term is used in full there
    assert 0.8 < c.worst_ratio < 1 and c.rel_l2 < 2e-3


def test_one_wrong_corner_pixel_fails_although_rel_l2_passes():
    """A halo bug that makes the bottom-right pixel read its left neighbour: all 96 channels wrong."""
    g = torch.Generator().manual_seed(1)
    T, H, W, C = 2, 256, 448, 96  # 22 M elements
    want = torch.randn(T, H, W, C, generator=g)
    got = want.to(torch.bfloat16)
    got[-1, -1, -1] = got[-1, -1, -2]
    c = measure(got, want)
    assert c.rel_l2 < 4e-3, c.rel_l2  # rel-L2 alone cannot see it ...
    assert c.n_bad > C // 2 and c.worst_index[:3] == (T - 1, H - 1, W - 1)  # ... the elementwise bound points at it
    with pytest.raises(AssertionError, match=r"exceed .* worst element at \(1, 255, 447, \d+\) of shape \(2, 256, 448, 96\)"):
        assert_close_bf16(got, want, "corner pixel")


def test_nan_and_rel_l2_failures_are_reported():
    want = torch.linspace(-2, 2, 4096).view(4, 8, 8, 16)
    got = want.to(torch.bfloat16)
    got[2, 5, 1, 7] = float("nan")
    with pytest.raises(AssertionError, match=r"1 of 4096 elements exceed .* at \(2, 5, 1, 7\)"):
        assert_close_bf16(got, want, "nan")
    scaled = want * (1 + 2 ** -8)  # within the elementwise bound everywhere, but rel-L2 3.9e-3 > 1e-3
    with pytest.raises(AssertionError, match=r"rel-L2 .* got -2\.0078"):
        assert_close_bf16(scaled, want, "drift", rel_l2=1e-3)


def test_fp32_result_is_not_modified_and_worst_value_is_its_own():
    """fp32 results (the head conv's planes, fp32 GEMM outputs, whole decodes) go through the same in-place arithmetic."""
    g = torch.Generator().manual_seed(2)
    want = torch.randn(3, 5, 9, 16, generator=g)
    got = want + 1e-3 * torch.randn(3, 5, 9, 16, generator=g)
    got[1, 4, 8, 3] += 0.5
    got_before, want_before = got.clone(), want.clone()
    c = measure(got, want)
    assert torch.equal(got, got_before) and torch.equal(want, want_before)
    assert c.worst_index == (1, 4, 8, 3) and c.n_bad >= 1
    assert c.got_at_worst == float(got[c.worst_index]) and c.want_at_worst == float(want[c.worst_index])
    with pytest.raises(AssertionError, match=f"got {float(got[1, 4, 8, 3]):.6g}, want {float(want[1, 4, 8, 3]):.6g}"):
        assert_close_bf16(got, want, "fp32")
    assert torch.equal(got, got_before)
