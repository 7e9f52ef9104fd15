"""Hopper-native (sm_90a) Wan2.1 VAE decode: drop-in for the reference's `sgm.models.wan_vae.WanVAE`
(sgm/models/wan_vae.py:619-666).  The module path contains "wan_vae" and the wrapper exposes `.model`
(an nn.Module), `.decode(list)` and `.encode(list)` exactly as SATVideoDiffusionEngine._init_first_stage /
decode_first_stage expect (diffusion_video.py:225-236, :298-309; SURVEY F11).

`WanVAE_` holds parameters under the reference's state_dict names (decoder.conv1.*, decoder.middle.N.*,
decoder.upsamples.N.*, decoder.head.*, conv2.*), so `load_state_dict(torch.load("Wan2.1_VAE.pth"), strict=False)`
fills it (decoder.* / conv2.* for decode, encoder.* / conv1.* for encode).

Compute path (all kernels of libscail_b200.so, activations channels-last bf16 [T,H,W,C]):
  whole-sequence causal 3x3x3 convs as wgmma implicit GEMMs with fused bias / residual epilogues,
  RMS_norm+SiLU as one pass, nearest-2x upsample as a gather, the time_conv frame interleave folded into the
  conv epilogue (incl. the reference's first-frame 'Rep' rule, wan_vae.py:105-131), per-frame mid-block
  attention (d=384) as GEMM -> row softmax -> GEMM, head conv writing clamped fp32 NCTHW directly.
"""
import torch
from torch import nn

from . import ops

MEAN = [-0.7571, -0.7089, -0.9113, 0.1075, -0.1745, 0.9653, -0.1517, 1.5508,
        0.4134, -0.0715, 0.5517, -0.3632, -0.1922, -0.9497, 0.2503, -0.2921]  # wan_vae.py:630-633
STD = [2.8184, 1.4541, 2.3275, 2.6558, 1.2196, 1.7708, 2.6052, 2.0743,
       3.2687, 2.1526, 2.8652, 1.5579, 1.6382, 1.1253, 2.8251, 1.9160]  # wan_vae.py:634-637


class CausalConv3d(nn.Conv3d):
    """Parameter holder with nn.Conv3d's weight/bias names and shapes (wan_vae.py:17-36)."""

    def packed(self):
        """[Cout, KT*KH*KW*Cin] bf16, tap-major / channel-minor; cached until the weight changes."""
        w = self.weight
        key = (w.data_ptr(), w._version, w.dtype, str(w.device))
        if getattr(self, "_pk_key", None) != key:
            self._pk = w.detach().permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()
            self._pk_key = key
        return self._pk


class _Conv2d(nn.Conv2d):
    def packed(self):
        w = self.weight
        key = (w.data_ptr(), w._version, w.dtype, str(w.device))
        if getattr(self, "_pk_key", None) != key:
            self._pk = w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()
            self._pk_key = key
        return self._pk


class RMS_norm(nn.Module):  # wan_vae.py:39-54
    def __init__(self, dim, channel_first=True, images=True, bias=False):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones((dim, 1, 1) if images else (dim, 1, 1, 1)))


class ResidualBlock(nn.Module):  # wan_vae.py:186-220
    def __init__(self, in_dim, out_dim, dropout=0.0):
        super().__init__()
        self.residual = nn.Sequential(RMS_norm(in_dim, images=False), nn.SiLU(), CausalConv3d(in_dim, out_dim, 3, padding=1),
                                      RMS_norm(out_dim, images=False), nn.SiLU(), nn.Dropout(dropout),
                                      CausalConv3d(out_dim, out_dim, 3, padding=1))
        self.shortcut = CausalConv3d(in_dim, out_dim, 1) if in_dim != out_dim else nn.Identity()

    def run(self, x):
        T, H, W, C = x.shape
        r = self.residual
        if isinstance(self.shortcut, nn.Identity):
            h = x
        else:
            sc = self.shortcut
            h = ops.gemm(x.view(-1, C), sc.weight.view(sc.weight.shape[0], C), sc.bias).view(T, H, W, -1)
        a = ops.rmsnorm_cl(x, r[0].gamma.view(-1), silu=True)
        y = ops.conv3d_cl(a, r[2].packed(), r[2].bias, 3, 3, 3, r[2].weight.shape[0])
        a = ops.rmsnorm_cl(y, r[3].gamma.view(-1), silu=True, out=a if a.shape == y.shape else None)
        return ops.conv3d_cl(a, r[6].packed(), r[6].bias, 3, 3, 3, r[6].weight.shape[0], residual=h, out=y)


class AttentionBlock(nn.Module):  # wan_vae.py:223-262
    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.norm = RMS_norm(dim)
        self.to_qkv = nn.Conv2d(dim, dim * 3, 1)
        self.proj = nn.Conv2d(dim, dim, 1)

    def run(self, x):
        T, H, W, C = x.shape
        L = H * W
        xn = ops.rmsnorm_cl(x, self.norm.gamma.view(-1), silu=False)
        wqkv, bqkv = self.to_qkv.weight.view(3 * C, C), self.to_qkv.bias
        qk = ops.gemm(xn.view(T * L, C), wqkv[:2 * C], bqkv[:2 * C])  # [T*L, 2C]
        out = torch.empty_like(x)
        s = torch.empty(L, L, device=x.device, dtype=torch.float32)
        p = torch.empty(L, L, device=x.device, dtype=torch.bfloat16)
        o = torch.empty(L, C, device=x.device, dtype=torch.bfloat16)
        wp = self.proj.weight.view(C, C)
        for t in range(T):  # one frame = one single-head attention over h*w tokens
            f = qk[t * L:(t + 1) * L]
            ops.gemm(f[:, :C], f[:, C:], None, out=s)                        # S = Q K^T (fp32)
            ops.softmax_rows(s, C ** -0.5, out=p)                            # softmax(S / sqrt(C))
            vt = ops.gemm(wqkv[2 * C:], xn.view(T * L, C)[t * L:(t + 1) * L], None)  # V^T = Wv Xn^T  [C, L]
            ops.gemm(p, vt, bqkv[2 * C:], out=o)                             # O = P V + b_v  (rows of P sum to 1)
            ops.gemm(o, wp, self.proj.bias, out=out.view(T * L, C)[t * L:(t + 1) * L], epilogue=ops.EPI_BIAS_RES,
                     residual=x.view(T * L, C)[t * L:(t + 1) * L])
        return out


class Resample(nn.Module):  # wan_vae.py:66-160
    def __init__(self, dim, mode):
        super().__init__()
        assert mode in ("upsample2d", "upsample3d", "downsample2d", "downsample3d")
        self.dim, self.mode = dim, mode
        if mode.startswith("upsample"):
            self.resample = nn.Sequential(nn.Upsample(scale_factor=(2.0, 2.0), mode="nearest-exact"),
                                          _Conv2d(dim, dim // 2, 3, padding=1))
            if mode == "upsample3d":
                self.time_conv = CausalConv3d(dim, dim * 2, (3, 1, 1), padding=(1, 0, 0))
        else:
            self.resample = nn.Sequential(nn.ZeroPad2d((0, 1, 0, 1)), _Conv2d(dim, dim, 3, stride=(2, 2)))
            if mode == "downsample3d":
                self.time_conv = CausalConv3d(dim, dim, (3, 1, 1), stride=(2, 1, 1), padding=(0, 0, 0))

    def run_down(self, x):
        """Encoder path (wan_vae.py:138-160): per-frame ZeroPad2d((0,1,0,1)) + 3x3 stride-2 conv, then for downsample3d
        the stride-2 time_conv over frames (2k-2, 2k-1, 2k) for k >= 1 while frame 0 bypasses it (first chunk only
        fills the cache, :146-148)."""
        T, H, W, C = x.shape
        c2 = self.resample[1]
        y = ops.conv3d_strided_cl(x, c2.packed(), c2.bias, 1, 3, 3, C, (T, H // 2, W // 2), sstride=2)
        if self.mode == "downsample3d" and T > 1:
            To = 1 + (T - 1) // 2
            z = torch.empty(To, H // 2, W // 2, C, device=x.device, dtype=torch.bfloat16)
            z[0].copy_(y[0])
            tc = self.time_conv
            ops.conv3d_strided_cl(y, tc.packed(), tc.bias, 3, 1, 1, C, (To - 1, H // 2, W // 2), tstride=2, toff=0, out=z[1:])
            y = z
        return y

    def run(self, x):
        if self.mode.startswith("downsample"):
            return self.run_down(x)
        T, H, W, C = x.shape
        if self.mode == "upsample3d" and T > 1:
            # frame 0 bypasses time_conv ('Rep'); frames 1.. form a fresh causal sequence whose two output
            # channel halves become frames 1+2i and 2+2i (wan_vae.py:105-137)
            y = torch.empty(1 + 2 * (T - 1), H, W, C, device=x.device, dtype=torch.bfloat16)
            y[0].copy_(x[0])
            tc = self.time_conv
            ops.conv3d_cl(x[1:], tc.packed(), tc.bias, 3, 1, 1, 2 * C, out=y[1:], fmul=2, ocols=C)
            x = y
        up = ops.upsample2x_cl(x)
        c2 = self.resample[1]
        return ops.conv3d_cl(up, c2.packed(), c2.bias, 1, 3, 3, C // 2)


class Encoder3d(nn.Module):  # wan_vae.py:265-366
    def __init__(self, dim=96, z_dim=32, dim_mult=(1, 2, 4, 4), num_res_blocks=2, attn_scales=(),
                 temperal_downsample=(False, True, True), dropout=0.0):
        super().__init__()
        if list(attn_scales):
            raise NotImplementedError("Wan2.1 VAE uses attn_scales=[]")
        dims = [dim * u for u in [1] + list(dim_mult)]
        self.conv1 = CausalConv3d(3, dims[0], 3, padding=1)
        downs = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            for _ in range(num_res_blocks):
                downs.append(ResidualBlock(in_dim, out_dim))
                in_dim = out_dim
            if i != len(dim_mult) - 1:
                downs.append(Resample(out_dim, "downsample3d" if temperal_downsample[i] else "downsample2d"))
        self.downsamples = nn.Sequential(*downs)
        self.middle = nn.Sequential(ResidualBlock(out_dim, out_dim), AttentionBlock(out_dim), ResidualBlock(out_dim, out_dim))
        self.head = nn.Sequential(RMS_norm(out_dim, images=False), nn.SiLU(), CausalConv3d(out_dim, z_dim, 3, padding=1))

    def conv1_packed(self):
        """[Cout, 27*8]: the 3 RGB input channels are zero-padded to 8 (TMA rows are 16-byte multiples)."""
        w = self.conv1.weight
        key = (w.data_ptr(), w._version, str(w.device))
        if getattr(self, "_c1_key", None) != key:
            wp = w.detach().permute(0, 2, 3, 4, 1)
            wp = torch.cat([wp, torch.zeros(*wp.shape[:-1], 5, device=w.device, dtype=w.dtype)], -1)
            self._c1 = wp.reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()
            self._c1_key = key
        return self._c1

    def run(self, x8):
        x = ops.conv3d_cl(x8, self.conv1_packed(), self.conv1.bias, 3, 3, 3, self.conv1.weight.shape[0])
        for m in self.downsamples:
            x = m.run(x)
        for m in self.middle:
            x = m.run(x)
        a = ops.rmsnorm_cl(x, self.head[0].gamma.view(-1), silu=True)
        hc = self.head[2]
        return ops.conv3d_cl(a, hc.packed(), hc.bias, 3, 3, 3, hc.weight.shape[0])


class Decoder3d(nn.Module):  # wan_vae.py:369-472
    def __init__(self, dim=96, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2, attn_scales=(),
                 temperal_upsample=(True, True, False), dropout=0.0):
        super().__init__()
        if list(attn_scales):
            raise NotImplementedError("Wan2.1 VAE uses attn_scales=[]")
        dims = [dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]
        self.conv1 = CausalConv3d(z_dim, dims[0], 3, padding=1)
        self.middle = nn.Sequential(ResidualBlock(dims[0], dims[0]), AttentionBlock(dims[0]), ResidualBlock(dims[0], dims[0]))
        ups = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            if i in (1, 2, 3):
                in_dim = in_dim // 2
            for _ in range(num_res_blocks + 1):
                ups.append(ResidualBlock(in_dim, out_dim))
                in_dim = out_dim
            if i != len(dim_mult) - 1:
                ups.append(Resample(out_dim, "upsample3d" if temperal_upsample[i] else "upsample2d"))
        self.upsamples = nn.Sequential(*ups)
        self.head = nn.Sequential(RMS_norm(out_dim, images=False), nn.SiLU(), CausalConv3d(out_dim, 3, 3, padding=1))

    def run(self, x):
        c1 = self.conv1
        x = ops.conv3d_cl(x, c1.packed(), c1.bias, 3, 3, 3, c1.weight.shape[0])
        for m in self.middle:
            x = m.run(x)
        for m in self.upsamples:
            x = m.run(x)
        a = ops.rmsnorm_cl(x, self.head[0].gamma.view(-1), silu=True)
        hc = self.head[2]
        return ops.conv3d_cl(a, hc.packed(), hc.bias, 3, 3, 3, 3, head=True)  # fp32 [3, T, H, W], clamped


class WanVAE_(nn.Module):
    """Decoder half of wan_vae.py:483-589 (same ctor kwargs)."""

    def __init__(self, dim=96, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2, attn_scales=(),
                 temperal_downsample=(False, True, True), dropout=0.0):
        super().__init__()
        self.z_dim = z_dim
        self.encoder = Encoder3d(dim, z_dim * 2, dim_mult, num_res_blocks, attn_scales, tuple(temperal_downsample), dropout)
        self.conv1 = CausalConv3d(z_dim * 2, z_dim * 2, 1)
        self.conv2 = CausalConv3d(z_dim, z_dim, 1)
        self.decoder = Decoder3d(dim, z_dim, dim_mult, num_res_blocks, attn_scales, tuple(temperal_downsample)[::-1], dropout)

    def decode(self, z, scale):
        """z [1,16,T,h,w]; scale = [mean, 1/std] (tensors).  Returns fp32 [1,3,1+4(T-1),8h,8w] in [-1,1]."""
        if not z.is_cuda:
            raise RuntimeError("scail_b200 has no CPU path: the VAE decode needs a CUDA (sm_90a) device")
        assert z.shape[0] == 1 and z.shape[1] == 16
        zb = z[0].to(torch.bfloat16).contiguous()
        mean = scale[0].to(device=z.device, dtype=torch.float32).contiguous()
        inv_std = scale[1].to(device=z.device, dtype=torch.float32).contiguous()
        x = ops.vae_latent_to_cl(zb, mean, inv_std)  # [T,h,w,16]
        T, h, w, C = x.shape
        c2 = self.conv2
        x = ops.gemm(x.view(-1, C), c2.weight.view(C, C), c2.bias).view(T, h, w, C)  # 1x1x1 conv2
        return self.decoder.run(x).unsqueeze(0)

    def encode(self, x, scale):
        """x [1,3,T,H,W] (T = 1 + 4k), values in [-1,1]; scale = [mean, 1/std].  Returns mu [1,16,1+k,H/8,W/8] fp32,
        (mu - mean) / std (wan_vae.py:516-542).  Whole-sequence causal convolutions; see Resample.run_down for the
        first-frame rule of the temporal downsampling."""
        if not x.is_cuda:
            raise RuntimeError("scail_b200 has no CPU path: the VAE encode needs a CUDA (sm_90a) device")
        assert x.shape[0] == 1 and x.shape[1] == 3
        _, _, T, H, W = x.shape
        x8 = torch.zeros(T, H, W, 8, device=x.device, dtype=torch.bfloat16)
        x8[..., :3] = x[0].permute(1, 2, 3, 0)
        y = self.encoder.run(x8)  # [T', h, w, 32]
        Tp, h, w, C = y.shape
        c1 = self.conv1
        y = ops.gemm(y.view(-1, C), c1.weight.view(C, C), c1.bias).view(Tp, h, w, C)
        mu = y[..., :self.z_dim].float().permute(3, 0, 1, 2)[None]
        mean = scale[0].to(device=x.device, dtype=torch.float32).view(1, -1, 1, 1, 1)
        inv_std = scale[1].to(device=x.device, dtype=torch.float32).view(1, -1, 1, 1, 1)
        return (mu - mean) * inv_std


class WanVAE:
    """Same surface as the reference wrapper (wan_vae.py:619-666)."""

    def __init__(self, z_dim=16, vae_pth=None, dtype=torch.bfloat16, device="cuda", **cfg):
        dtype = eval(dtype) if not isinstance(dtype, torch.dtype) else dtype
        self.dtype, self.device = dtype, device
        self.mean = torch.tensor(MEAN, dtype=torch.float32, device=device)
        self.std = torch.tensor(STD, dtype=torch.float32, device=device)
        self.scale = [self.mean, 1.0 / self.std]
        self.model = WanVAE_(z_dim=z_dim, **cfg)
        if vae_pth is not None:
            # the reference's load is mandatory and strict (wan_vae.py:607-616: load_state_dict(..., assign=True)); the
            # parameter names are identical, so anything missing or unexpected is a wrong / partial checkpoint
            self.model.load_state_dict(torch.load(vae_pth, map_location="cpu"), strict=True)
        else:
            import warnings
            warnings.warn("scail_b200.wan_vae.WanVAE: vae_pth is None -> RANDOM weights (tests / benchmarks only)")
        self.model = self.model.eval().requires_grad_(False).to(device).to(torch.bfloat16)

    def encode(self, videos):
        """videos: list of [3, T, H, W] tensors (wan_vae.py:648-657)."""
        return torch.cat([self.model.encode(u.unsqueeze(0), self.scale).float() for u in videos], dim=0)

    def decode(self, zs):
        return torch.cat([self.model.decode(u.unsqueeze(0), self.scale).float().clamp_(-1, 1) for u in zs], dim=0)
