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

Chunked decode / encode (`chunk_frames=k`): the same kernels over k latent frames at a time, so activation memory
does not grow with the video length (the reference's WanVAE_.decode / encode run 1 latent frame per chunk with a
feat_cache, wan_vae.py:516-568).  Every causal conv keeps the last <= KT-1 frames of its input stream in a
_ChunkState and reads them as the causal history of the next chunk (scail_conv3d_cl_hist); everything else is per
frame or per pixel.  The result is bit-identical to the whole-sequence path.
"""
import torch
from torch import nn

from . import ops

MEAN = [-0.7571, -0.7089, -0.9113, 0.1075, -0.1745, 0.9653, -0.1517, 1.5508,
        0.4134, -0.0715, 0.5517, -0.3632, -0.1922, -0.9497, 0.2503, -0.2921]  # wan_vae.py:630-633
STD = [2.8184, 1.4541, 2.3275, 2.6558, 1.2196, 1.7708, 2.6052, 2.0743,
       3.2687, 2.1526, 2.8652, 1.5579, 1.6382, 1.1253, 2.8251, 1.9160]  # wan_vae.py:634-637


def check_chunk_frames(k):
    """None (whole sequence) or an int >= 1 (latent frames per chunk)."""
    if k is None:
        return None
    if isinstance(k, bool) or int(k) != k or k < 1:
        raise ValueError(f"chunk_frames must be None or an integer >= 1, got {k!r}")
    return int(k)


def chunk_ranges(n, k):
    """Latent frame ranges [(a, b), ...] of a chunked run over n latent frames, k per chunk (the last may be shorter)."""
    k = check_chunk_frames(k)
    return [(a, min(a + k, n)) for a in range(0, n, k)]


def frame_range(a, b, up):
    """Frames [p0, p1) of a stage `up` times longer in time that latent frames [a, b) map to.  Latent frame 0 is frame 0,
    latent frame j >= 1 is frames up*(j-1)+1 .. up*j (the first-frame rule: T latent frames <-> 1 + up*(T-1) frames).
    up = 4 gives the pixel frames: chunk 0 holds 1 + 4(k-1) of them, every later chunk 4k."""
    return (0 if a == 0 else up * (a - 1) + 1, up * (b - 1) + 1)


class _History:
    """The last <= n frames of one causal conv's input stream.  The buffer is allocated once per call and keeps its
    address, so the conv's TMA descriptor for it is reused from chunk to chunk."""

    def __init__(self, n):
        self.n, self.buf, self.count = n, None, 0

    def frames(self):
        return None if self.count == 0 else self.buf[self.n - self.count:]

    def keep(self, x):
        f = x.shape[0]
        if f == 0:
            return
        if self.buf is None:
            self.buf = torch.empty((self.n,) + tuple(x.shape[1:]), device=x.device, dtype=x.dtype)
        if f >= self.n:
            self.buf.copy_(x[f - self.n:])
        else:  # n == 2, f == 1: shift the newer frame down (frames 0 and 1 do not overlap)
            self.buf[:self.n - f].copy_(self.buf[f:])
            self.buf[self.n - f:].copy_(x)
        self.count = min(self.n, self.count + f)


class _ChunkState:
    """Per-call state of a chunked decode / encode: one _History per causal conv (keyed by the conv module), and
    whether the current chunk is the first one (it holds frame 0 of every stage, where the 'Rep' rules apply)."""

    def __init__(self):
        self.first = True
        self._h = {}

    def frames(self, conv):
        h = self._h.get(conv)
        return None if h is None else h.frames()

    def keep(self, conv, x, n=2):
        if conv not in self._h:
            self._h[conv] = _History(n)
        self._h[conv].keep(x)


def _hist(st, conv):
    return None if st is None else st.frames(conv)


def _keep(st, conv, x, n=2):
    """Record the tail of conv's input; call it before x's buffer is reused (ResidualBlock.run overwrites `a`)."""
    if st is not None:
        st.keep(conv, x, n)


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

    def run(self, x, st=None):
        T, H, W, C = x.shape
        r = self.residual
        if isinstance(self.shortcut, nn.Identity):
            h = x
        else:
            sc = self.shortcut
            h = ops.gemm(x.view(-1, C), sc.weight.view(sc.weight.shape[0], C), sc.bias).view(T, H, W, -1)
        a = ops.rmsnorm_cl(x, r[0].gamma.view(-1), silu=True)
        y = ops.conv3d_cl(a, r[2].packed(), r[2].bias, 3, 3, 3, r[2].weight.shape[0], hist=_hist(st, r[2]))
        _keep(st, r[2], a)  # before the next norm overwrites a
        a = ops.rmsnorm_cl(y, r[3].gamma.view(-1), silu=True, out=a if a.shape == y.shape else None)
        y = ops.conv3d_cl(a, r[6].packed(), r[6].bias, 3, 3, 3, r[6].weight.shape[0], residual=h, out=y, hist=_hist(st, r[6]))
        _keep(st, r[6], a)
        return y


class AttentionBlock(nn.Module):  # wan_vae.py:223-262
    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.norm = RMS_norm(dim)
        self.to_qkv = nn.Conv2d(dim, dim * 3, 1)
        self.proj = nn.Conv2d(dim, dim, 1)

    def run(self, x, st=None):  # per frame: no state across chunks
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

    def run_down(self, x, st=None):
        """Encoder path (wan_vae.py:138-160): per-frame ZeroPad2d((0,1,0,1)) + 3x3 stride-2 conv, then for downsample3d
        the stride-2 time_conv over frames (2k-2, 2k-1, 2k) for k >= 1 while frame 0 bypasses it (first chunk only
        fills the cache, :146-148).  In a later chunk of a chunked run, output j reads local frames 2j-1 .. 2j+1: toff -1,
        with the previous chunk's last frame as a 1-frame history (the reference's x[:, :, -1:] cache, :151-157)."""
        T, H, W, C = x.shape
        c2 = self.resample[1]
        y = ops.conv3d_strided_cl(x, c2.packed(), c2.bias, 1, 3, 3, C, (T, H // 2, W // 2), sstride=2)
        if self.mode != "downsample3d":
            return y
        tc = self.time_conv
        if st is not None and not st.first:
            z = ops.conv3d_strided_cl(y, tc.packed(), tc.bias, 3, 1, 1, C, (T // 2, H // 2, W // 2), tstride=2, toff=-1,
                                      hist=st.frames(tc))
            _keep(st, tc, y, n=1)
            return z
        if T > 1:
            To = 1 + (T - 1) // 2
            z = torch.empty(To, H // 2, W // 2, C, device=x.device, dtype=torch.bfloat16)
            z[0].copy_(y[0])
            ops.conv3d_strided_cl(y, tc.packed(), tc.bias, 3, 1, 1, C, (To - 1, H // 2, W // 2), tstride=2, toff=0, out=z[1:])
            _keep(st, tc, y, n=1)
            y = z
        else:
            _keep(st, tc, y, n=1)
        return y

    def run(self, x, st=None):
        if self.mode.startswith("downsample"):
            return self.run_down(x, st)
        T, H, W, C = x.shape
        tc = getattr(self, "time_conv", None)
        if self.mode == "upsample3d" and st is not None and not st.first:
            # a later chunk: all its frames continue the causal sequence that started at frame 1
            y = torch.empty(2 * T, H, W, C, device=x.device, dtype=torch.bfloat16)
            ops.conv3d_cl(x, tc.packed(), tc.bias, 3, 1, 1, 2 * C, out=y, fmul=2, ocols=C, hist=st.frames(tc))
            _keep(st, tc, x)
            x = y
        elif self.mode == "upsample3d" and T > 1:
            # frame 0 bypasses time_conv ('Rep'); frames 1.. form a fresh causal sequence whose two output
            # channel halves become frames 1+2i and 2+2i (wan_vae.py:105-137)
            y = torch.empty(1 + 2 * (T - 1), H, W, C, device=x.device, dtype=torch.bfloat16)
            y[0].copy_(x[0])
            ops.conv3d_cl(x[1:], tc.packed(), tc.bias, 3, 1, 1, 2 * C, out=y[1:], fmul=2, ocols=C)
            _keep(st, tc, x[1:])
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

    def time_factor(self):
        """Pixel frames per latent frame after the first (4 for Wan2.1)."""
        return 2 ** sum(isinstance(m, Resample) and m.mode == "downsample3d" for m in self.downsamples)

    def run(self, x8, st=None):
        x = ops.conv3d_cl(x8, self.conv1_packed(), self.conv1.bias, 3, 3, 3, self.conv1.weight.shape[0],
                          hist=_hist(st, self.conv1))
        _keep(st, self.conv1, x8)
        for m in self.downsamples:
            x = m.run(x, st)
        for m in self.middle:
            x = m.run(x, st)
        a = ops.rmsnorm_cl(x, self.head[0].gamma.view(-1), silu=True)
        hc = self.head[2]
        y = ops.conv3d_cl(a, hc.packed(), hc.bias, 3, 3, 3, hc.weight.shape[0], hist=_hist(st, hc))
        _keep(st, hc, a)
        return y


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

    def scale_factors(self):
        """(frames per latent frame after the first, spatial factor): (4, 8) for Wan2.1."""
        ups = [m for m in self.upsamples if isinstance(m, Resample)]
        return 2 ** sum(m.mode == "upsample3d" for m in ups), 2 ** len(ups)

    def run(self, x, st=None, out=None, out_frame_offset=0):
        """x [T,h,w,z_dim] -> fp32 [3, T', H, W], clamped; or written into frames out_frame_offset.. of out [3, *, H, W]."""
        c1 = self.conv1
        x0 = x
        x = ops.conv3d_cl(x, c1.packed(), c1.bias, 3, 3, 3, c1.weight.shape[0], hist=_hist(st, c1))
        _keep(st, c1, x0)
        for m in self.middle:
            x = m.run(x, st)
        for m in self.upsamples:
            x = m.run(x, st)
        a = ops.rmsnorm_cl(x, self.head[0].gamma.view(-1), silu=True)
        hc = self.head[2]
        y = ops.conv3d_cl(a, hc.packed(), hc.bias, 3, 3, 3, 3, head=True, out=out, out_frame_offset=out_frame_offset,
                          hist=_hist(st, hc))  # fp32 [3, T, H, W], clamped
        _keep(st, hc, a)
        return y


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

    def decode(self, z, scale, chunk_frames=None):
        """z [1,16,T,h,w]; scale = [mean, 1/std] (tensors).  Returns fp32 [1,3,1+4(T-1),8h,8w] in [-1,1].
        chunk_frames=None decodes the whole sequence at once; k >= 1 decodes latent frames [c*k, (c+1)*k) per chunk
        (bit-identical result, activation memory independent of T)."""
        k = check_chunk_frames(chunk_frames)
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
        if k is None:
            return self.decoder.run(x).unsqueeze(0)
        up, s = self.decoder.scale_factors()
        out = torch.empty(3, frame_range(0, T, up)[1], s * h, s * w, device=z.device, dtype=torch.float32)
        st = _ChunkState()
        for a, b in chunk_ranges(T, k):  # the head conv writes each chunk's frames straight into `out`
            self.decoder.run(x[a:b], st, out=out, out_frame_offset=frame_range(a, b, up)[0])
            st.first = False
        return out.unsqueeze(0)

    def encode(self, x, scale, chunk_frames=None):
        """x [1,3,T,H,W] (T = 1 + 4k), values in [-1,1]; scale = [mean, 1/std].  Returns mu [1,16,1+k,H/8,W/8] fp32,
        (mu - mean) / std (wan_vae.py:516-542).  Whole-sequence causal convolutions; see Resample.run_down for the
        first-frame rule of the temporal downsampling.  chunk_frames=k >= 1 encodes the pixel frames of k latent frames
        per chunk (1 + 4(k-1), then 4k; k = 1 is the reference's 1, 4, 4, ... split) with a bit-identical result."""
        k = check_chunk_frames(chunk_frames)
        if not x.is_cuda:
            raise RuntimeError("scail_b200 has no CPU path: the VAE encode needs a CUDA (sm_90a) device")
        assert x.shape[0] == 1 and x.shape[1] == 3
        _, _, T, H, W = x.shape
        if k is None:
            x8 = torch.zeros(T, H, W, 8, device=x.device, dtype=torch.bfloat16)
            x8[..., :3] = x[0].permute(1, 2, 3, 0)
            y = self.encoder.run(x8)  # [T', h, w, 32]
        else:
            up = self.encoder.time_factor()
            if (T - 1) % up:
                raise ValueError(f"chunked encode needs 1 + {up}*n frames, got {T}")
            st, ys = _ChunkState(), []
            for a, b in chunk_ranges(1 + (T - 1) // up, k):
                p0, p1 = frame_range(a, b, up)
                x8 = torch.zeros(p1 - p0, H, W, 8, device=x.device, dtype=torch.bfloat16)
                x8[..., :3] = x[0, :, p0:p1].permute(1, 2, 3, 0)
                ys.append(self.encoder.run(x8, st))
                st.first = False
            y = torch.cat(ys)
        Tp, h, w, C = y.shape
        c1 = self.conv1
        y = ops.gemm(y.view(-1, C), c1.weight.view(C, C), c1.bias).view(Tp, h, w, C)
        mu = y[..., :self.z_dim].float().permute(3, 0, 1, 2)[None]
        mean = scale[0].to(device=x.device, dtype=torch.float32).view(1, -1, 1, 1, 1)
        inv_std = scale[1].to(device=x.device, dtype=torch.float32).view(1, -1, 1, 1, 1)
        return (mu - mean) * inv_std


class WanVAE:
    """Same surface as the reference wrapper (wan_vae.py:619-666)."""

    def __init__(self, z_dim=16, vae_pth=None, dtype=torch.bfloat16, device="cuda", chunk_frames=None, **cfg):
        """chunk_frames: default of .decode / .encode (None = whole sequence, k >= 1 = k latent frames per chunk)."""
        dtype = eval(dtype) if not isinstance(dtype, torch.dtype) else dtype
        self.dtype, self.device = dtype, device
        self.chunk_frames = check_chunk_frames(chunk_frames)
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

    def encode(self, videos, chunk_frames=None):
        """videos: list of [3, T, H, W] tensors (wan_vae.py:648-657).  chunk_frames: None = the constructor's default."""
        k = self.chunk_frames if chunk_frames is None else check_chunk_frames(chunk_frames)
        return torch.cat([self.model.encode(u.unsqueeze(0), self.scale, chunk_frames=k).float() for u in videos], dim=0)

    def decode(self, zs, chunk_frames=None):
        """zs: list of [16, T, h, w] latents.  chunk_frames: None = the constructor's default."""
        k = self.chunk_frames if chunk_frames is None else check_chunk_frames(chunk_frames)
        return torch.cat([self.model.decode(u.unsqueeze(0), self.scale, chunk_frames=k).float().clamp_(-1, 1) for u in zs],
                         dim=0)
