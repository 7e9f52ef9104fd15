"""Chunked (temporally tiled) Wan2.1 VAE decode / encode on the GPU.

A conv with a causal history must compute, bit for bit, what the same conv computes on cat(history, x) for the frames
of x: the history only changes where the t < 0 boxes are fetched from, never the taps, channel slices or their order.
So chunked decode / encode must equal the whole-sequence path under torch.equal, and their activation memory must not
grow with the number of frames."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm())


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(torch.bfloat16).cuda()


def pack(w):
    return w.permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1).contiguous()


def random_vae(dim, seed):
    from scail_b200.wan_vae import WanVAE
    torch.manual_seed(seed)
    vae = WanVAE(dim=dim)
    with torch.no_grad():
        for n, p in vae.model.named_parameters():
            if p.dim() >= 2 and p.numel() > p.shape[0] and "gamma" not in n:
                p.copy_(torch.randn_like(p) / p[0].numel() ** 0.5)
            elif "gamma" in n:
                p.copy_(1 + 0.1 * torch.randn_like(p))
            else:
                p.copy_(0.02 * torch.randn_like(p))
    return vae


# (T, H, W, Cin, Cout, taps): conv3d_kernel<16>, <96>, <192> (also 3x1x1), row-tile kernel with one / two 96-wide N blocks
CONV_CASES = [(3, 8, 16, 16, 16, (3, 3, 3)), (3, 8, 24, 64, 96, (3, 3, 3)), (2, 10, 20, 96, 192, (3, 3, 3)),
              (3, 8, 8, 128, 256, (3, 1, 1)), (2, 6, 128, 96, 96, (3, 3, 3)), (2, 5, 256, 192, 192, (3, 3, 3))]


@pytest.mark.parametrize("T_hist", [0, 1, 2])
@pytest.mark.parametrize("T,H,W,Cin,Cout,k", CONV_CASES)
def test_conv_with_history_equals_conv_over_concatenation(T, H, W, Cin, Cout, k, T_hist):
    from scail_b200 import ops
    x, hist = rnd(T, H, W, Cin, seed=1), rnd(T_hist, H, W, Cin, seed=2)
    w2 = pack(rnd(Cout, Cin, *k, seed=3, scale=(Cin * k[0] * k[1] * k[2]) ** -0.5))
    b, res = rnd(Cout, seed=4), rnd(T, H, W, Cout, seed=5)
    xc = torch.cat([hist, x]).contiguous()
    got = ops.conv3d_cl(x, w2, b, *k, Cout, hist=hist)
    want = ops.conv3d_cl(xc, w2, b, *k, Cout)[T_hist:]
    assert torch.equal(got, want)
    got_r = ops.conv3d_cl(x, w2, b, *k, Cout, residual=res, hist=hist)
    want_r = ops.conv3d_cl(xc, w2, b, *k, Cout, residual=torch.cat([torch.zeros_like(res[:T_hist]), res]))[T_hist:]
    assert torch.equal(got_r, want_r)
    if T_hist:  # the history is really read: frame 0 differs from zero padding
        assert not torch.equal(got[0], ops.conv3d_cl(x, w2, b, *k, Cout)[0])


@pytest.mark.parametrize("T_hist", [1, 2])
def test_time_conv_interleave_with_history(T_hist):
    """upsample3d time_conv: 3x1x1, two channel halves written as frames 2t and 2t+1 (fmul=2)."""
    from scail_b200 import ops
    T, H, W, C = 3, 8, 16, 64
    x, hist = rnd(T, H, W, C, seed=1), rnd(T_hist, H, W, C, seed=2)
    w2, b = pack(rnd(2 * C, C, 3, 1, 1, seed=3, scale=(3 * C) ** -0.5)), rnd(2 * C, seed=4)
    got = torch.empty(2 * T, H, W, C, device="cuda", dtype=torch.bfloat16)
    ops.conv3d_cl(x, w2, b, 3, 1, 1, 2 * C, out=got, fmul=2, ocols=C, hist=hist)
    want = torch.empty(2 * (T_hist + T), H, W, C, device="cuda", dtype=torch.bfloat16)
    ops.conv3d_cl(torch.cat([hist, x]).contiguous(), w2, b, 3, 1, 1, 2 * C, out=want, fmul=2, ocols=C)
    assert torch.equal(got, want[2 * T_hist:])


def test_strided_time_conv_with_one_frame_history():
    """downsample3d time_conv of a later encoder chunk: stride 2, toff -1, the previous chunk's last frame as history."""
    from scail_b200 import ops
    T, H, W, C = 8, 6, 10, 64
    x, hist = rnd(T, H, W, C, seed=1), rnd(1, H, W, C, seed=2)
    w2, b = pack(rnd(C, C, 3, 1, 1, seed=3, scale=(3 * C) ** -0.5)), rnd(C, seed=4)
    got = ops.conv3d_strided_cl(x, w2, b, 3, 1, 1, C, (T // 2, H, W), tstride=2, toff=-1, hist=hist)
    want = ops.conv3d_strided_cl(torch.cat([hist, x]).contiguous(), w2, b, 3, 1, 1, C, (T // 2, H, W), tstride=2, toff=0)
    assert torch.equal(got, want)


@pytest.mark.parametrize("W", [24, 256])  # conv3d_kernel<16> and the N=16 row-tile head
def test_head_writes_frames_at_offset(W):
    from scail_b200 import ops
    T, H, C, T_hist, T_total, off = 2, 5, 96, 2, 7, 3
    x, hist = rnd(T, H, W, C, seed=1), rnd(T_hist, H, W, C, seed=2)
    w2, b = pack(rnd(3, C, 3, 3, 3, seed=3, scale=0.04)), rnd(3, seed=4)
    big = torch.full((3, T_total, H, W), 7.0, device="cuda")
    got = ops.conv3d_cl(x, w2, b, 3, 3, 3, 3, head=True, out=big, out_frame_offset=off, hist=hist)
    assert got is big
    want = ops.conv3d_cl(torch.cat([hist, x]).contiguous(), w2, b, 3, 3, 3, 3, head=True)[:, T_hist:]
    assert torch.equal(big[:, off:off + T], want)
    assert bool((big[:, :off] == 7.0).all()) and bool((big[:, off + T:] == 7.0).all())


def test_decode_chunked_matches_whole_sequence_and_reference_golden():
    from scail_b200.wan_vae import WanVAE
    g = torch.load(os.path.join(GOLD, "vae_small.pt"))
    vae = WanVAE(dim=g["dim"])
    vae.model.load_state_dict(g["state_dict"], strict=False)
    vae.model = vae.model.to("cuda").to(torch.bfloat16)
    z = g["z"][0].cuda()
    whole = vae.decode([z])
    for k in (1, 2, 3):
        got = vae.decode([z], chunk_frames=k)
        assert got.shape == whole.shape and torch.equal(got, whole), k
    e = rel(vae.decode([z], chunk_frames=1), g["out"])
    print("chunked VAE decode relL2 vs reference fp32:", e)
    assert e < 2e-2


def test_decode_chunked_matches_whole_sequence_full_width():
    """dim=96 on a latent 16 wide: the 96-channel stages are 128 px wide, so the row-tile kernels run with histories."""
    vae = random_vae(96, seed=1)
    z = rnd(16, 5, 16, 16, seed=9)
    whole = vae.decode([z])
    assert whole.shape == (1, 3, 17, 128, 128) and bool(torch.isfinite(whole).all())
    for k in (1, 2, 3):
        assert torch.equal(vae.decode([z], chunk_frames=k), whole), k
    vae.chunk_frames = 2  # the constructor default (YAML first_stage_config.params.chunk_frames) is used by .decode(list)
    assert torch.equal(vae.decode([z]), whole)


def test_encode_chunked_matches_whole_sequence_and_reference_golden():
    from scail_b200.wan_vae import WanVAE
    g = torch.load(os.path.join(GOLD, "vae_encode_small.pt"))
    vae = WanVAE(dim=g["dim"])
    vae.model.load_state_dict(g["state_dict"], strict=False)
    vae.model = vae.model.to("cuda").to(torch.bfloat16)
    video = g["video"][0].cuda()
    whole = vae.encode([video])
    for k in (1, 2, 3):
        got = vae.encode([video], chunk_frames=k)
        assert got.shape == whole.shape and torch.equal(got, whole), k
    e = rel(vae.encode([video], chunk_frames=1), g["mu"])
    print("chunked VAE encode relL2 vs reference fp32:", e)
    assert e < 2e-2


def test_encode_chunked_matches_whole_sequence_full_width():
    vae = random_vae(96, seed=2)
    g = torch.Generator().manual_seed(3)
    video = (torch.rand(3, 21, 32, 128, generator=g) * 2 - 1).cuda()  # 6 latent frames; full-res stage 128 px wide
    whole = vae.encode([video])
    assert whole.shape == (1, 16, 6, 4, 16) and bool(torch.isfinite(whole).all())
    for k in (1, 2, 3, 4):
        assert torch.equal(vae.encode([video], chunk_frames=k), whole), k
    with pytest.raises(ValueError):
        vae.encode([video[:, :20]], chunk_frames=1)


def test_chunked_decode_memory_does_not_grow_with_frames():
    vae = random_vae(96, seed=3)
    m = vae.model

    def peak(z, k):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = m.decode(z[None], vae.scale, chunk_frames=k)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, out.numel() * out.element_size()

    z3, z9 = rnd(16, 3, 16, 16, seed=4), rnd(16, 9, 16, 16, seed=5)
    peak(z3, 1)  # warm-up: packed weights are cached on the first call
    p3, o3 = peak(z3, 1)
    p9, o9 = peak(z9, 1)
    pw, _ = peak(z9, None)
    print(f"peak activation bytes: chunked T=3 {p3 / 2**20:.1f} MiB, T=9 {p9 / 2**20:.1f} MiB; whole T=9 {pw / 2**20:.1f} MiB")
    assert p9 - p3 <= (o9 - o3) + z9.numel() * z9.element_size() + 16 * 2**20
    assert pw >= 2 * p9
