"""BENCH COMPARISON ARM ONLY — the reference's op chain on the PyTorch *library* path, on the GPU, in bf16.

SURVEY.md §2.2 / §8(d): the reference has no hand-written kernel on the hot path; what it launches on an H100 is
`F.linear` (cuBLASLt), `F.layer_norm`, `F.scaled_dot_product_attention` (flash / cuDNN), `F.gelu`, elementwise torch ops,
and cuDNN `conv3d` for the VAE.  The UNMODIFIED reference cannot travel to the GPU box (no /root/reference there, and it
needs deepspeed / omegaconf / pytorch_lightning), so `bench.py --impl torchlib` and the `library_baseline` key time THIS
restatement of its op sequence — one bf16 rounding per op, a separate bias add after RowParallelLinear, RoPE as
`t*cos + rotate_half(t)*sin` in bf16 — against the same weights (the product model's own nn.Parameters, no copy) and the
same inputs.  It is "the bar to beat on the same box".  Nothing under scail_b200/ imports this module and it launches none
of the library's kernels.

Reference lines restated (paths relative to /root/reference):
  DiffusionTransformer.forward            dit_video_crossattn_sc_xc.py:1452-1587
  ImagePatchEmbeddingMixin                :99-130        Rotary3DPositionEmbeddingMixin.attention_fn   :653-757
  AdaLNMixin.layer_forward / attention_forward / cross_attention_forward                               :1009-1203
  FinalLayerMixin.final_forward           :818-835       attention_fn_default   sat/transformer_defaults.py:47-79
  ColumnParallelLinear / RowParallelLinear sat/mpu/layers.py:230-243, 425-444 (Row: F.linear(x, W) then `+ bias`)
  mlp_forward_default                     sat/transformer_defaults.py:163-176
  VanillaCFG / RFSampler.sampler_step     guiders.py:41-57, sampling.py:950-963
  WanVAE_.decode and its blocks           sgm/models/wan_vae.py:17-262, 369-472, 544-568
"""
import math

import torch
import torch.nn.functional as F

from scail_b200 import rope as _rope  # host-side table builder only (bit-identical to the reference's ctor tables)


def _rotate_half(x):  # dit_video_crossattn_sc_xc.py:336-340 (interleaved pairs)
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack((-x2, x1), -1).flatten(-2)


def _rmsnorm(x, w, eps=1e-6):  # :61-68: fp32 math, one cast back
    xf = x.float()
    return (w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))).to(x.dtype)


def _ln(x, w=None, b=None, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def _heads(x, h):
    b, n, d = x.shape
    return x.view(b, n, h, d // h).permute(0, 2, 1, 3)


def _merge(x):
    b, h, n, d = x.shape
    return x.permute(0, 2, 1, 3).reshape(b, n, h * d)


def _row_linear(x, lin):  # RowParallelLinear: matmul, then bias as a second bf16 op (sat/mpu/layers.py:436-443)
    y = F.linear(x, lin.weight)
    return y + lin.bias if lin.bias is not None else y


def _col_linear(x, lin):
    return F.linear(x, lin.weight, lin.bias)


def _timestep_embedding(t, dim, max_period=10000):  # sgm/modules/diffusionmodules/util.py:207-231
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float64, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], -1).float()


@torch.no_grad()
def dit_forward(model, x, timesteps, context, ref_concat, concat_smpl_render, image_clip_features):
    """Library-path forward of a scail_b200.dit.DiffusionTransformer's weights.  x [b,t,16,h,w]; returns [b,t,16,h,w] bf16."""
    bf = torch.bfloat16
    dev = x.device
    b, t, _, h, w = x.shape
    H = model.num_attention_heads
    d = model.hidden_size
    x = x.to(bf)
    rep = lambda a: a.to(bf).repeat(b // a.shape[0], *([1] * (a.dim() - 1)))
    images = torch.cat([x, torch.zeros(b, t, 4, h, w, dtype=bf, device=dev)], 2)          # :1468,1503
    ref = torch.cat([rep(ref_concat), torch.ones(b, 1, 4, h, w, dtype=bf, device=dev)], 2)  # :1483-1486
    pose = torch.cat([rep(concat_smpl_render), torch.ones(b, t, 4, h // 2, w // 2, dtype=bf, device=dev)], 2)
    # ---- embeddings (:1505-1555) ----
    te = model.text_embedding
    text = te[2](te[1](te[0](context.to(bf))))
    clip = model.clip_proj.proj(rep(image_clip_features))
    t_emb = _timestep_embedding(timesteps.to(dev), model.time_freq_dim).to(bf)
    emb = model.time_embed(t_emb)
    adaln = model.adaln_projection(emb)
    # ---- patch embed: Conv3d k=s=(1,2,2) (:99-130) ----
    pe = model.mixins["patch_embed"]
    conv = lambda u, c: c(u.permute(0, 2, 1, 3, 4)).flatten(2).transpose(1, 2)  # b c t h w -> b (t h w) c
    hid = torch.cat([conv(torch.cat([ref, images], 1), pe.proj), conv(pose, pe.proj_pose)], 1)
    cos, sin = _rope.build_tables(dev, d // H, t, h // 2, w // 2)
    cos, sin = cos.to(bf), sin.to(bf)  # `.to(t.dtype)` (:553-554)
    ad = model.mixins["adaln_layer"]
    for l, layer in enumerate(model.transformer.layers):
        mod = adaln.unflatten(1, (6, d)) + ad.adaLN_modulations[l]
        sh_a, sc_a, g_a, sh_m, sc_m, g_m = mod.chunk(6, 1)
        # self attention (:1031-1036, 1058-1105)
        a_in = _ln(hid) * (1 + sc_a) + sh_a
        q, k, v = _col_linear(a_in, layer.attention.query_key_value).chunk(3, -1)
        q = _heads(_rmsnorm(q, ad.query_layernorm_list[l].weight), H)
        k = _heads(_rmsnorm(k, ad.key_layernorm_list[l].weight), H)
        v = _heads(v, H)
        q = q * cos + _rotate_half(q) * sin
        k = k * cos + _rotate_half(k) * sin
        o = _merge(F.scaled_dot_product_attention(q, k, v))
        del q, k, v
        hid = hid + g_a * _row_linear(o, layer.attention.dense)
        # cross attention (:1039-1042, 1107-1203)
        pl = layer.post_cross_attention_layernorm
        c_in = _ln(hid, pl.weight, pl.bias)
        ca = layer.cross_attention
        q = _heads(_rmsnorm(_col_linear(c_in, ca.query), ad.cross_query_layernorm_list[l].weight), H)
        kt, vt = _col_linear(text, ca.key_value).chunk(2, -1)
        kt = _rmsnorm(kt, ad.cross_key_layernorm_list[l].weight)
        kc, vc = _col_linear(clip, ad.clip_feature_key_value_list[l]).chunk(2, -1)
        kc = _rmsnorm(kc, ad.clip_feature_key_layernorm_list[l].weight)
        o = _merge(F.scaled_dot_product_attention(q, _heads(kt, H), _heads(vt, H)))
        o = o + _merge(F.scaled_dot_product_attention(q, _heads(kc, H), _heads(vc, H)))
        del q
        hid = hid + _row_linear(o, ca.dense)
        # MLP (:1045-1050)
        m_in = _ln(hid) * (1 + sc_m) + sh_m
        hmid = F.gelu(_col_linear(m_in, layer.mlp.dense_h_to_4h), approximate="tanh")
        hid = hid + g_m * _row_linear(hmid, layer.mlp.dense_4h_to_h)
        del hmid, a_in, c_in, m_in, o
    fl = model.mixins["final_layer"]
    shift, scale = (emb.unsqueeze(1) + fl.adaLN_modulation).chunk(2, 1)
    out = fl.linear(_ln(hid) * (1 + scale) + shift)
    n_ref, n_seq = h * w // 4, t * h * w // 4
    out = out[:, n_ref:n_ref + n_seq].reshape(b, t, h // 2, w // 2, 1, 2, 2, 16)
    return out.permute(0, 1, 4, 7, 2, 5, 3, 6).reshape(b, t, 16, h, w)  # 'b (t h w) (o p q c) -> b (t o) c (h p) (w q)'


@torch.no_grad()
def sampler_step(model, x, sigma, next_sigma, cond, uc, scale=4.0):
    """Reference sampler step on library kernels: CFG batch-2 forward, `u + s(c - u)`, Euler (fp32 latent)."""
    x2 = torch.cat([x, x], 0)
    ts = torch.full((2,), float(sigma) * 1000.0, device=x.device, dtype=torch.float32)
    ctx = torch.cat([uc["crossattn"], cond["crossattn"]], 0)
    v = dit_forward(model, x2, ts, ctx, cond["ref_concat"], cond["concat_smpl_render"], cond["image_clip_features"]).float()
    vu, vc = v.chunk(2)
    return x + (float(next_sigma) - float(sigma)) * (vu + scale * (vc - vu))


# ------------------------------------------------------------------------------------------------------------------
# Wan2.1 VAE decode on cuDNN conv3d (bf16, channels_last_3d), whole-sequence form of the reference's chunked decode
# ------------------------------------------------------------------------------------------------------------------


def _cconv(x, conv):  # CausalConv3d (wan_vae.py:17-36)
    w = conv.weight
    kt, kh, kw = w.shape[2:]
    return F.conv3d(F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0)), w, conv.bias)


def _vrms(x, gamma):  # RMS_norm (:39-54), channel-first
    return F.normalize(x, dim=1) * (x.shape[1] ** 0.5) * gamma.view(1, -1, *([1] * (x.dim() - 2)))


def _vres(blk, x):  # ResidualBlock (:186-220)
    hsc = _cconv(x, blk.shortcut) if not isinstance(blk.shortcut, torch.nn.Identity) else x
    r = blk.residual
    y = _cconv(F.silu(_vrms(x, r[0].gamma)), r[2])
    y = _cconv(F.silu(_vrms(y, r[3].gamma)), r[6])
    return y + hsc


def _vattn(blk, x):  # AttentionBlock (:223-262)
    b, c, t, h, w = x.shape
    y = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
    y = _vrms(y, blk.norm.gamma)
    qkv = F.conv2d(y, blk.to_qkv.weight, blk.to_qkv.bias).reshape(b * t, 1, 3 * c, h * w).permute(0, 1, 3, 2)
    q, k, v = qkv.chunk(3, -1)
    o = F.scaled_dot_product_attention(q.contiguous(), k.contiguous(), v.contiguous()).squeeze(1).permute(0, 2, 1).reshape(b * t, c, h, w)
    o = F.conv2d(o, blk.proj.weight, blk.proj.bias)
    return o.reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4) + x


def _vup(blk, x):  # Resample upsample2d / upsample3d (:101-160)
    b, c, t, h, w = x.shape
    if blk.mode == "upsample3d" and t > 1:
        y = _cconv(x[:, :, 1:], blk.time_conv).reshape(b, 2, c, t - 1, h, w)
        y = torch.stack((y[:, 0], y[:, 1]), 3).reshape(b, c, 2 * (t - 1), h, w)
        x = torch.cat([x[:, :, :1], y], 2)
        t = x.shape[2]
    y = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
    y = F.interpolate(y.float(), scale_factor=(2.0, 2.0), mode="nearest-exact").to(x.dtype)
    conv = blk.resample[1]
    y = F.conv2d(y, conv.weight, conv.bias, padding=1)
    return y.reshape(b, t, c // 2, 2 * h, 2 * w).permute(0, 2, 1, 3, 4)


@torch.no_grad()
def vae_decode(vae, z):
    """vae: scail_b200.wan_vae.WanVAE (its parameters are used as-is); z [16,T,h,w] -> fp32 [1,3,1+4(T-1),8h,8w]."""
    from scail_b200.wan_vae import AttentionBlock, Resample, ResidualBlock
    m = vae.model
    bf = torch.bfloat16
    mean, inv_std = vae.scale[0].view(1, 16, 1, 1, 1), vae.scale[1].view(1, 16, 1, 1, 1)
    x = (z[None].float() / inv_std + mean).to(bf).contiguous(memory_format=torch.channels_last_3d)
    x = _cconv(x, m.conv2)
    dec = m.decoder
    x = _cconv(x, dec.conv1)
    for blk in list(dec.middle) + list(dec.upsamples):
        if isinstance(blk, ResidualBlock):
            x = _vres(blk, x)
        elif isinstance(blk, AttentionBlock):
            x = _vattn(blk, x)
        elif isinstance(blk, Resample):
            x = _vup(blk, x)
        else:
            raise TypeError(type(blk))
    x = F.silu(_vrms(x, dec.head[0].gamma))
    return _cconv(x, dec.head[2]).float().clamp_(-1, 1)
