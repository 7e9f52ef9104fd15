"""GPU parity of the Wan2.1 VAE decode path through the C ABI:
 (a) against the golden vector produced by the UNMODIFIED reference (tests/golden/vae_small.pt: dim=16 variant,
     latent [1,16,3,8,8] -> [1,3,9,64,64], fp32 chunked decode with the feature cache),
 (b) single-op checks of the wgmma implicit-GEMM causal conv against F.conv3d in fp32.
Tolerance: output is in [-1,1] after clamp; rel-L2 vs the fp32 reference <= 2e-2 over ~40 bf16 layers,
per-op rel-L2 <= 4e-3 (one bf16 rounding)."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm())


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(torch.bfloat16).cuda()


@pytest.mark.parametrize("T,H,W,Cin,Cout,k", [(3, 8, 16, 64, 96, (3, 3, 3)), (2, 10, 20, 96, 192, (3, 3, 3)),
                                              (4, 16, 16, 16, 384, (3, 3, 3)), (3, 8, 8, 128, 256, (3, 1, 1)),
                                              (2, 24, 40, 192, 96, (1, 3, 3)), (2, 16, 16, 384, 384, (3, 3, 3)),
                                              # W >= 128 and Cout % 96 == 0 -> row-tile kernel (taps = shifted smem views)
                                              (2, 6, 128, 96, 96, (3, 3, 3)), (2, 5, 256, 192, 192, (3, 3, 3)),
                                              (1, 4, 160, 64, 96, (3, 3, 3)), (2, 7, 384, 192, 96, (1, 3, 3)),
                                              (3, 3, 128, 384, 384, (3, 3, 3))])
def test_conv3d_cl_vs_torch(T, H, W, Cin, Cout, k):
    from scail_b200 import ops
    x = rnd(T, H, W, Cin, seed=1)
    w = rnd(Cout, Cin, *k, seed=2, scale=(Cin * k[0] * k[1] * k[2]) ** -0.5)
    b = rnd(Cout, seed=3)
    res = rnd(T, H, W, Cout, seed=4)
    w2 = w.permute(0, 2, 3, 4, 1).reshape(Cout, -1).contiguous()
    got = ops.conv3d_cl(x, w2, b, *k, Cout)
    got_r = ops.conv3d_cl(x, w2, b, *k, Cout, residual=res)
    xin = x.float().permute(3, 0, 1, 2)[None]
    xin = F.pad(xin, (k[2] // 2, k[2] // 2, k[1] // 2, k[1] // 2, k[0] - 1, 0))
    want = F.conv3d(xin, w.float(), b.float())[0].permute(1, 2, 3, 0)
    torch.cuda.synchronize()
    assert rel(got, want) < 4e-3, rel(got, want)
    assert rel(got_r, want + res.float()) < 4e-3


def test_time_conv_interleave_and_head():
    from scail_b200 import ops
    T, H, W, C = 3, 8, 16, 64
    x = rnd(T, H, W, C, seed=1)
    w = rnd(2 * C, C, 3, 1, 1, seed=2, scale=(3 * C) ** -0.5)
    b = rnd(2 * C, seed=3)
    out = torch.zeros(2 * T, H, W, C, device="cuda", dtype=torch.bfloat16)
    ops.conv3d_cl(x, w.permute(0, 2, 3, 4, 1).reshape(2 * C, -1).contiguous(), b, 3, 1, 1, 2 * C, out=out, fmul=2, ocols=C)
    xin = F.pad(x.float().permute(3, 0, 1, 2)[None], (0, 0, 0, 0, 2, 0))
    y = F.conv3d(xin, w.float(), b.float())  # [1, 2C, T, H, W]
    y = y.reshape(1, 2, C, T, H, W)
    y = torch.stack((y[:, 0], y[:, 1]), 3).reshape(1, C, 2 * T, H, W)[0].permute(1, 2, 3, 0)
    assert rel(out, y) < 4e-3
    # head: Cout = 3, fp32 planes, clamp
    wh, bh = rnd(3, C, 3, 3, 3, seed=5, scale=0.05), rnd(3, seed=6)
    got = ops.conv3d_cl(x, wh.permute(0, 2, 3, 4, 1).reshape(3, -1).contiguous(), bh, 3, 3, 3, 3, head=True)
    xin = F.pad(x.float().permute(3, 0, 1, 2)[None], (1, 1, 1, 1, 2, 0))
    want = F.conv3d(xin, wh.float(), bh.float())[0].clamp(-1, 1)
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert float((got - want).abs().max()) < 2e-2
    # same head conv at W >= 128: row-tile kernel instantiated with N = 16
    x2 = rnd(2, 5, 256, 96, seed=7)
    wh2, bh2 = rnd(3, 96, 3, 3, 3, seed=8, scale=0.04), rnd(3, seed=9)
    got2 = ops.conv3d_cl(x2, wh2.permute(0, 2, 3, 4, 1).reshape(3, -1).contiguous(), bh2, 3, 3, 3, 3, head=True)
    xin2 = F.pad(x2.float().permute(3, 0, 1, 2)[None], (1, 1, 1, 1, 2, 0))
    want2 = F.conv3d(xin2, wh2.float(), bh2.float())[0].clamp(-1, 1)
    assert got2.shape == want2.shape and float((got2 - want2).abs().max()) < 2e-2


def test_vae_elementwise():
    from scail_b200 import ops
    for C in (16, 96, 192, 384):
        x, g = rnd(5, 7, 9, C, seed=C), rnd(C, seed=1) * 0.1 + 1
        want = F.normalize(x.float(), dim=-1) * C ** 0.5 * g.float()
        assert rel(ops.rmsnorm_cl(x, g, silu=False), want) < 4e-3
        assert rel(ops.rmsnorm_cl(x, g, silu=True), F.silu(want)) < 4e-3
    x = rnd(3, 5, 6, 32, seed=2)
    up = ops.upsample2x_cl(x)
    want = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=(2.0, 2.0), mode="nearest-exact").permute(0, 2, 3, 1)
    assert torch.equal(up.float(), want)
    s = torch.randn(70, 333, device="cuda") * 5
    assert rel(ops.softmax_rows(s, 0.3), torch.softmax(s * 0.3, -1)) < 4e-3
    z = rnd(16, 3, 4, 5, seed=3)
    mean, inv = torch.randn(16, device="cuda"), torch.rand(16, device="cuda") + 0.5
    want = (z.float() / inv.view(16, 1, 1, 1) + mean.view(16, 1, 1, 1)).permute(1, 2, 3, 0)
    assert rel(ops.vae_latent_to_cl(z, mean, inv), want) < 4e-3


def test_vae_decode_against_reference_golden():
    from scail_b200.wan_vae import WanVAE
    g = torch.load(os.path.join(GOLD, "vae_small.pt"))
    vae = WanVAE(dim=g["dim"])
    missing, unexpected = vae.model.load_state_dict(g["state_dict"], strict=False)
    assert not unexpected and all(k.startswith(("encoder.", "conv1.")) for k in missing)
    vae.model = vae.model.to("cuda").to(torch.bfloat16)
    out = vae.decode([g["z"][0].cuda()])
    torch.cuda.synchronize()
    assert out.shape == g["out"].shape and out.dtype == torch.float32
    e = rel(out, g["out"])
    print("VAE decode relL2 vs reference fp32:", e, "max abs", float((out.cpu() - g["out"]).abs().max()))
    assert e < 2e-2


def test_vae_decode_full_width_against_oracle():
    """dim=96 (the real width) on a tiny latent; oracle in fp32 on the GPU."""
    from oracle import vae_oracle as V
    from scail_b200.wan_vae import WanVAE
    torch.manual_seed(0)
    vae = WanVAE(dim=96)
    with torch.no_grad():
        for n, p in vae.model.named_parameters():
            if p.dim() >= 2 and p.numel() > p.shape[0] and "gamma" not in n:
                p.copy_(torch.randn_like(p) / p[0].numel() ** 0.5)
            elif "gamma" in n:
                p.copy_(1 + 0.1 * torch.randn_like(p))
            else:
                p.copy_(0.02 * torch.randn_like(p))
    sd = {k: v.float().cuda() for k, v in vae.model.state_dict().items()}
    z = rnd(16, 2, 4, 4, seed=9)
    V_mean, V_std = torch.tensor(V.MEAN), torch.tensor(V.STD)
    with torch.device("cuda"):
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        want = V.decode(sd, z[None].float())
    got = vae.decode([z])
    e = rel(got, want)
    print("full-width VAE relL2 vs oracle:", e)
    assert e < 2e-2


def test_strided_convs_vs_torch():
    """Encoder Resample pieces: 3x3 stride-2 conv behind ZeroPad2d((0,1,0,1)) and the 3x1x1 stride-2 time_conv."""
    from scail_b200 import ops
    T, H, W, C = 3, 12, 20, 64
    x = rnd(T, H, W, C, seed=1)
    w, b = rnd(C, C, 3, 3, seed=2, scale=(9 * C) ** -0.5), rnd(C, seed=3)
    got = ops.conv3d_strided_cl(x, w.permute(0, 2, 3, 1).reshape(C, -1).contiguous(), b, 1, 3, 3, C, (T, H // 2, W // 2), sstride=2)
    want = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), w.float(), b.float(), stride=2).permute(0, 2, 3, 1)
    assert rel(got, want) < 4e-3
    T = 9
    x = rnd(T, 6, 10, C, seed=4)
    wt, bt = rnd(C, C, 3, 1, 1, seed=5, scale=(3 * C) ** -0.5), rnd(C, seed=6)
    got = ops.conv3d_strided_cl(x, wt.permute(0, 2, 3, 4, 1).reshape(C, -1).contiguous(), bt, 3, 1, 1, C, ((T - 1) // 2, 6, 10),
                                tstride=2, toff=0)
    want = F.conv3d(x.float().permute(3, 0, 1, 2)[None], wt.float(), bt.float(), stride=(2, 1, 1))[0].permute(1, 2, 3, 0)
    assert rel(got, want) < 4e-3


def test_vae_encode_against_reference_golden():
    """SURVEY §8f rank 2: encode path vs the golden produced by the UNMODIFIED reference (chunked 1+4+4 frames)."""
    from scail_b200.wan_vae import WanVAE
    g = torch.load(os.path.join(GOLD, "vae_encode_small.pt"))
    vae = WanVAE(dim=g["dim"])
    missing, unexpected = vae.model.load_state_dict(g["state_dict"], strict=False)
    assert not unexpected and all(k.startswith(("decoder.", "conv2.")) for k in missing)
    vae.model = vae.model.to("cuda").to(torch.bfloat16)
    mu = vae.encode([g["video"][0].cuda()])
    torch.cuda.synchronize()
    assert mu.shape == g["mu"].shape and mu.dtype == torch.float32
    e = rel(mu, g["mu"])
    print("VAE encode relL2 vs reference fp32:", e)
    assert e < 2e-2


def test_conv_fused_norm_epilogue_and_full_width_decode_at_128():
    """Row-tile conv with the optional fused RMS_norm+SiLU second output (Cout == 96; measured slower end to end than the
    separate norm pass, so wan_vae.py does not use it yet), then the dim=96 decoder on a latent whose 96-channel stage
    is 128 px wide so the row-tile kernels (incl. the N=16 head) run at the real channel widths."""
    from oracle import vae_oracle as V
    from scail_b200 import ops
    from scail_b200.wan_vae import WanVAE
    T, H, W, C = 2, 4, 128, 96
    x, res = rnd(T, H, W, C, seed=1), rnd(T, H, W, C, seed=2)
    w, b, g = rnd(C, C, 3, 3, 3, seed=3, scale=(27 * C) ** -0.5), rnd(C, seed=4), rnd(C, seed=5) * 0.1 + 1
    w2 = w.permute(0, 2, 3, 4, 1).reshape(C, -1).contiguous()
    out, a = ops.conv3d_cl(x, w2, b, 3, 3, 3, C, residual=res, norm_gamma=g)
    xin = F.pad(x.float().permute(3, 0, 1, 2)[None], (1, 1, 1, 1, 2, 0))
    want = F.conv3d(xin, w.float(), b.float())[0].permute(1, 2, 3, 0) + res.float()
    want_a = F.silu(F.normalize(want, dim=-1) * C ** 0.5 * g.float())
    assert rel(out, want) < 4e-3 and rel(a, want_a) < 6e-3
    none_out, a2 = ops.conv3d_cl(x, w2, b, 3, 3, 3, C, norm_gamma=g, want_raw=False)
    want2 = want - res.float()
    assert none_out is None and rel(a2, F.silu(F.normalize(want2, dim=-1) * C ** 0.5 * g.float())) < 6e-3
    torch.manual_seed(1)
    vae = WanVAE(dim=96)
    with torch.no_grad():
        for n, p in vae.model.named_parameters():
            if p.dim() >= 2 and p.numel() > p.shape[0] and "gamma" not in n:
                p.copy_(torch.randn_like(p) / p[0].numel() ** 0.5)
            elif "gamma" in n:
                p.copy_(1 + 0.1 * torch.randn_like(p))
            else:
                p.copy_(0.02 * torch.randn_like(p))
    sd = {k: v.float().cuda() for k, v in vae.model.state_dict().items()}
    z = rnd(16, 2, 16, 16, seed=9)  # -> 5 x 128 x 128
    with torch.device("cuda"):
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        want = V.decode(sd, z[None].float())
    got = vae.decode([z])
    e = rel(got, want)
    print("full-width VAE @128px relL2 vs oracle:", e)
    assert got.shape == want.shape and e < 2e-2
